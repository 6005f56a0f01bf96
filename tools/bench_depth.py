#!/usr/bin/env python
"""Times colour + depth rendering, forward and backward, two ways on the same seeded scenes:
  fused     render_views_with_depth: the depth map is a fourth channel of the colour compositor;
  two_pass  render_views + render_depth_views: the reference's route, a second rasterization over per-view copies
            of the Gaussians.
configs[1] shape by default (re10k-like, 256x256, 2 context views x 3 Gaussians per pixel = 393 216 Gaussians,
SH degree 4).  Random dL/dC and dL/dD, eager calls, a pool of scenes larger than L2, three alternating rounds of
--steps steps per route, CUDA events, median.  Prints one JSON line with both rates, their ratio, the card name and
its power limit.

    python tools/bench_depth.py [--mode depth] [--views 1] [--steps 100] [--dump-outputs DIR]

--dump-outputs DIR writes the colour and depth images of the last fused step (float32 .npy) for output-for-output
comparisons between builds.  Nothing else is written.
"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

GAUSS_KEYS = ("means", "covariances", "harmonics", "opacities")


def gpu_identity(index: int) -> dict:
    """Card name and power limit: part of every number this tool reports."""
    out = {"card": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return out


def step(d, d_img, d_dep, image, mode, fused):
    """One colour + depth forward and backward; returns (colour, depth, gradients)."""
    from pixelsplat_b200.decoder import render_views, render_views_with_depth
    from pixelsplat_b200.decoder.cuda_splatting import render_depth_views
    leaves = [d[k] for k in GAUSS_KEYS]
    cam = (d["extrinsics"][None], d["intrinsics"][None], d["near"][None], d["far"][None], image)
    bg = torch.zeros((1, d["extrinsics"].shape[0], 3), device=d["means"].device)
    if fused:
        img, depth = render_views_with_depth(*cam, bg, *leaves, mode=mode)
    else:
        img = render_views(*cam, bg, *leaves)
        depth = render_depth_views(*cam, leaves[0], leaves[1], leaves[3], mode=mode)
    grads = torch.autograd.grad((img, depth), leaves, (d_img, d_dep))
    return img, depth, grads


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="depth", choices=["depth", "disparity", "relative_disparity", "log"])
    ap.add_argument("--views", type=int, default=1, help="target views per call (one scene)")
    ap.add_argument("--image", type=int, default=256)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--pool", type=int, default=4, help="distinct scenes cycled (> L2 in total)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_depth.py needs a CUDA device: pixelsplat_b200 has no CPU path")
    from pixelsplat_b200 import rasterizer, synthetic
    dev = torch.device("cuda", 0)
    image, V = (args.image, args.image), args.views
    pool = []
    for i in range(args.pool):
        sc = synthetic.scene_re10k_like(seed=i, image_hw=image, context_views=2, gaussians_per_pixel=3,
                                        sh_degree=4, target_views=V)
        d = dict(extrinsics=sc.extrinsics, intrinsics=sc.intrinsics, near=sc.near, far=sc.far, means=sc.means[None],
                 covariances=sc.covariances[None], harmonics=sc.harmonics[None], opacities=sc.opacities[None])
        d = {k: v.contiguous().float().to(dev) for k, v in d.items()}
        for k in GAUSS_KEYS:
            d[k].requires_grad_(True)
        pool.append(d)
    g = torch.Generator().manual_seed(7)
    d_img = torch.randn((1, V, 3, *image), generator=g).to(dev)
    d_dep = torch.randn((1, V, *image), generator=g).to(dev)

    rasterizer.set_capacity_check("sync")           # sizes the binning buffers of every scene
    for fused in (True, False):
        for i in range(args.warmup):
            step(pool[i % args.pool], d_img, d_dep, image, args.mode, fused)
    rasterizer.set_capacity_check("deferred")       # verified when each backward starts
    torch.cuda.synchronize()
    rates = {True: [], False: []}
    last = None
    for _ in range(3):
        for fused in (True, False):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(args.steps):
                out = step(pool[i % args.pool], d_img, d_dep, image, args.mode, fused)
            b.record()
            torch.cuda.synchronize()
            rates[fused].append(args.steps * V / (a.elapsed_time(b) * 1e-3))
            if fused:
                last = out
    fused_v, two_v = statistics.median(rates[True]), statistics.median(rates[False])
    line = {"metric": "colour+depth fwd+bwd", "mode": args.mode, "views_per_call": V, "image": list(image),
            "gaussians": int(pool[0]["means"].shape[1]), "fused": fused_v, "two_pass": two_v,
            "ratio": fused_v / two_v, "unit": "views/s", "rounds": {"fused": rates[True], "two_pass": rates[False]},
            "how": "eager calls, random dL/dC and dL/dD, 3 alternating rounds of --steps steps per route, median; "
                   "fused = render_views_with_depth, two_pass = render_views + render_depth_views"}
    line.update(gpu_identity(0))
    if args.dump_outputs:
        import numpy as np
        out_dir = Path(args.dump_outputs)
        out_dir.mkdir(parents=True, exist_ok=True)
        np.save(out_dir / "image.npy", last[0].detach().float().cpu().numpy())
        np.save(out_dir / "depth.npy", last[1].detach().float().cpu().numpy())
    print(json.dumps(line))


if __name__ == "__main__":
    main()
