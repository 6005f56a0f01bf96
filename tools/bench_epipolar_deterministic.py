#!/usr/bin/env python
"""Times the EpipolarTransformer's forward + backward with torch.use_deterministic_algorithms off and on (the
fixed-order d(feature map) of ps_epipolar_attention_backward_deterministic), on the same seeded inputs.  configs[2]
shapes: features [b, v, 128, 256, 256] -> 64 x 64 rays, 32 samples, 4 heads, 10 octaves, two layers.  Eager calls,
three alternating rounds of --steps steps per mode, CUDA events, median.  Under the flag torch also fills every
torch.empty (fill_uninitialized_memory, on by default): "on" is measured with that fill, "on_nofill" without it.
A torch.profiler pass per mode gives the per-kernel device times of one step.  Prints one JSON line: ms per step
per mode, the per-kernel times, the deterministic workspace per layer backward, the longest cell list (slots that
share one bilinear cell), the card name and its power limit.

    python tools/bench_epipolar_deterministic.py [--shapes 1x2,7x2,1x3] [--steps 10]

Nothing is written.
"""
import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from bench_depth import gpu_identity  # noqa: E402

MODES = ("off", "on", "on_nofill")


def set_mode(mode):
    torch.use_deterministic_algorithms(mode != "off")
    torch.utils.deterministic.fill_uninitialized_memory = mode != "on_nofill"


def build(b, v, hw, dev):
    from pixelsplat_b200 import synthetic
    from pixelsplat_b200.encoder import EpipolarTransformer, EpipolarTransformerCfg, ImageSelfAttentionCfg
    torch.manual_seed(0)
    cfg = EpipolarTransformerCfg(ImageSelfAttentionCfg(4, 10, 2, 4, 128, 128, 256), 10, 2, 4, 32, 128, 256, 4)
    enc = EpipolarTransformer(cfg, 128, num_context_views=v).to(dev)
    g = torch.Generator().manual_seed(1234)
    feats = torch.randn(b, v, 128, hw, hw, generator=g).to(dev).requires_grad_(True)
    ext = torch.eye(4).repeat(b, v, 1, 1)
    for i in range(v):
        ext[:, i, 0, 3] = float(i) / max(v - 1, 1)           # the train_step rig: views along x
    ext = ext.to(dev)
    k = synthetic.intrinsics_re10k(v)[None].repeat(b, 1, 1, 1).to(dev)
    near_v, far_v = synthetic.bounds_from_baseline(1.0, hw, hw, 3.0 * hw, 0.5)
    near, far = torch.full((b, v), near_v, device=dev), torch.full((b, v), far_v, device=dev)
    wgt = torch.randn(b, v, 128, hw, hw, generator=g).to(dev)
    return enc, (feats, ext, k, near, far), wgt


def step(enc, inputs, wgt):
    enc.zero_grad(set_to_none=True)
    inputs[0].grad = None
    out, _ = enc(*inputs)
    (out * wgt).sum().backward()


def longest_cell_list(enc, inputs, S):
    """Slots per bilinear cell of the first layer's sampling (the kernel's cell key, restated in torch)."""
    feats, ext, k, near, far = inputs
    b, v = feats.shape[:2]
    with torch.no_grad():
        h = enc.downscaler(feats.flatten(0, 1)).shape[-1] if enc.downscaler is not None else feats.shape[-1]
        geom = enc.epipolar_sampler.geometry((h, h), ext, k, near, far)
    seg, valid = geom.segments, geom.valid.bool()
    ov = v - 1
    u = (torch.arange(S, device=seg.device, dtype=torch.float32) + 0.5) / S
    sx = seg[..., None, 0] + u * (seg[..., None, 2] - seg[..., None, 0])
    sy = seg[..., None, 1] + u * (seg[..., None, 3] - seg[..., None, 1])
    bx = torch.floor(sx * h - 0.5).clamp(-2, h + 1)
    by = torch.floor(sy * h - 0.5).clamp(-2, h + 1)
    vi = torch.arange(v, device=seg.device)[:, None]
    o = torch.arange(ov, device=seg.device)[None, :]
    m = torch.arange(b, device=seg.device)[:, None, None] * v + torch.where(o < vi, o, o + 1)[None]
    key = (m[..., None, None] * (h + 1) + by + 1) * (h + 1) + bx + 1
    ok = valid[..., None] & (bx >= -1) & (bx < h) & (by >= -1) & (by < h)
    counts = torch.bincount(key[ok].long().flatten(), minlength=b * v * (h + 1) ** 2)
    return {"longest": int(counts.max()), "mean_nonempty": float(counts[counts > 0].float().mean()),
            "slots_with_record": int(ok.sum()), "slots": int(ok.numel()), "grid": [h, h]}


def kernel_times(enc, inputs, wgt):
    """Per-kernel device time of one step, in ms, for the kernels of the epipolar attention and the largest others."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(enc, inputs, wgt)
        torch.cuda.synchronize()
    rows = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            rows[e.key] = (t / 1e3, e.count)
    epi = {k[:120]: {"ms": round(t, 4), "calls": c} for k, (t, c) in rows.items() if "k_epi" in k}
    top = sorted(((t, k) for k, (t, c) in rows.items() if "k_epi" not in k), reverse=True)[:8]
    return {"epipolar_kernels": epi, "top_other": {k[:120]: round(t, 4) for t, k in top},
            "total_ms": round(sum(t for t, _ in rows.values()), 3)}


def bench_shape(args, b, v, dev):
    from pixelsplat_b200 import _lib
    enc, inputs, wgt = build(b, v, args.hw, dev)
    for mode in MODES:
        set_mode(mode)
        for _ in range(args.warmup):
            step(enc, inputs, wgt)
    torch.cuda.synchronize()
    ms = {m: [] for m in MODES}
    for _ in range(3):
        for mode in MODES:
            set_mode(mode)
            a, c = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.steps):
                step(enc, inputs, wgt)
            c.record()
            torch.cuda.synchronize()
            ms[mode].append(a.elapsed_time(c) / args.steps)
    kernels = {}
    for mode in MODES:
        set_mode(mode)
        kernels[mode] = kernel_times(enc, inputs, wgt)
    set_mode("off")
    h = args.hw // 4
    desc = _lib.EpipolarDesc(b, v, h, h, 32, 128, 4, 20)
    med = {m: statistics.median(r) for m, r in ms.items()}
    return {"batch": b, "views": v, "ms_per_step": med, "rounds": ms,
            "ratio_on": med["on"] / med["off"], "ratio_on_nofill": med["on_nofill"] / med["off"],
            "workspace_bytes_per_layer_backward": _lib.epipolar_backward_workspace_bytes(desc),
            "cell_lists": longest_cell_list(enc, inputs, 32), "kernels_one_step": kernels,
            "peak_gib": torch.cuda.max_memory_allocated() / 2 ** 30}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1x2,7x2,1x3", help="batch x views, comma-separated")
    ap.add_argument("--hw", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_epipolar_deterministic.py needs a CUDA device: pixelsplat_b200 has no CPU path")
    import os
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    dev = torch.device("cuda", 0)
    flag, fill = torch.are_deterministic_algorithms_enabled(), torch.utils.deterministic.fill_uninitialized_memory
    results = []
    try:
        for s in args.shapes.split(","):
            b, v = (int(x) for x in s.split("x"))
            torch.cuda.reset_peak_memory_stats()
            results.append(bench_shape(args, b, v, dev))
    finally:
        torch.use_deterministic_algorithms(flag)
        torch.utils.deterministic.fill_uninitialized_memory = fill
    line = {"metric": "EpipolarTransformer fwd+bwd, torch.use_deterministic_algorithms off / on",
            "features_hw": args.hw, "unit": "ms/step", "results": results,
            "how": "eager forward + (out * w).sum().backward(), 3 alternating rounds of --steps steps per mode, median; "
                   "on = deterministic flag with torch's fill of uninitialised memory, on_nofill = without it; "
                   "kernel times from one torch.profiler step per mode"}
    line.update(gpu_identity(0))
    print(json.dumps(line))


if __name__ == "__main__":
    main()
