#!/usr/bin/env python
"""Times the rasterizer's colour forward + backward with torch.use_deterministic_algorithms off and on (the library's
fixed-order composite backward, include/pixelsplat_b200.h option "deterministic"), on the same seeded scenes.
configs[1] shape by default (re10k-like, 256x256, 2 context views x 3 Gaussians per pixel = 393 216 Gaussians, SH
degree 4).  Random dL/dC, eager calls, a pool of scenes larger than L2, three alternating rounds of --steps steps per
mode, CUDA events, median.  Under the flag torch also fills every torch.empty (fill_uninitialized_memory, on by
default); the "on" rate is measured with that fill and, separately, without it.  Prints one JSON line: views/s per
mode and views-per-call, the ratios, the backward scratch bytes of both modes, the card name and its power limit.

    python tools/bench_deterministic.py [--views 1,4] [--steps 50] [--dump-outputs DIR]

--dump-outputs DIR writes the gradients of one deterministic step (first scene, first --views entry; float32 .npy)
for bit-for-bit comparisons between builds.  Nothing else is written.
"""
import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from bench_depth import GAUSS_KEYS, gpu_identity  # noqa: E402

MODES = ("off", "on", "on_nofill")


def step(d, d_img, image):
    """One colour forward and backward; returns the gradients of the Gaussians."""
    from pixelsplat_b200.decoder import render_views
    leaves = [d[k] for k in GAUSS_KEYS]
    cam = (d["extrinsics"][None], d["intrinsics"][None], d["near"][None], d["far"][None], image)
    bg = torch.zeros((1, d["extrinsics"].shape[0], 3), device=d["means"].device)
    img = render_views(*cam, bg, *leaves)
    return torch.autograd.grad(img, leaves, d_img)


def set_mode(mode):
    torch.use_deterministic_algorithms(mode != "off")
    torch.utils.deterministic.fill_uninitialized_memory = mode != "on_nofill"


def scratch_bytes(P, V, image):
    """Backward scratch of the shape as the benchmark ran it (its binning capacity), option off and on."""
    from pixelsplat_b200 import _lib, rasterizer
    dev = torch.cuda.current_device()
    capacity = rasterizer._capacity_hint[(dev, 1, V, P, *image)]
    desc = _lib.RasterDesc(1, V, P, 25, 4, _lib.PS_SH_3M, _lib.PS_COV_3X3, *image, 0, 0, capacity, 0, 0)
    out = {"instance_capacity": capacity}
    for mode in (0, 1):
        _lib.set_option("deterministic", mode)
        out["on" if mode else "off"] = _lib.sizes(desc).backward_bytes
    _lib.set_option("deterministic", 0)
    return out


def bench_views(args, V, image, dev):
    from pixelsplat_b200 import rasterizer, synthetic
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
    d_img = torch.randn((1, V, 3, *image), generator=torch.Generator().manual_seed(7)).to(dev)
    rasterizer.set_capacity_check("sync")           # sizes the binning buffers of every scene
    for mode in MODES:
        set_mode(mode)
        for i in range(args.warmup):
            step(pool[i % args.pool], d_img, image)
    rasterizer.set_capacity_check("deferred")       # verified when each backward starts
    torch.cuda.synchronize()
    rates = {m: [] for m in MODES}
    for _ in range(3):
        for mode in MODES:
            set_mode(mode)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(args.steps):
                step(pool[i % args.pool], d_img, image)
            b.record()
            torch.cuda.synchronize()
            rates[mode].append(args.steps * V / (a.elapsed_time(b) * 1e-3))
    grads = None
    if args.dump_outputs:
        set_mode("on")
        grads = step(pool[0], d_img, image)
    set_mode("off")
    med = {m: statistics.median(r) for m, r in rates.items()}
    res = {"views_per_call": V, "off": med["off"], "on": med["on"], "on_nofill": med["on_nofill"],
           "ratio_on": med["on"] / med["off"], "ratio_on_nofill": med["on_nofill"] / med["off"], "rounds": rates,
           "backward_scratch_bytes": scratch_bytes(int(pool[0]["means"].shape[1]), V, image)}
    return res, grads


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", default="1,4", help="target views per call (one scene), comma-separated")
    ap.add_argument("--image", type=int, default=256)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--pool", type=int, default=4, help="distinct scenes cycled (> L2 in total)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_deterministic.py needs a CUDA device: pixelsplat_b200 has no CPU path")
    dev = torch.device("cuda", 0)
    image = (args.image, args.image)
    flag, fill = torch.are_deterministic_algorithms_enabled(), torch.utils.deterministic.fill_uninitialized_memory
    results, dumped = [], None
    try:
        for V in (int(v) for v in args.views.split(",")):
            res, grads = bench_views(args, V, image, dev)
            results.append(res)
            dumped = dumped or grads
    finally:
        torch.use_deterministic_algorithms(flag)
        torch.utils.deterministic.fill_uninitialized_memory = fill
    line = {"metric": "colour fwd+bwd, torch.use_deterministic_algorithms off / on", "image": list(image),
            "unit": "views/s", "results": results,
            "how": "eager render_views + autograd.grad, random dL/dC, 3 alternating rounds of --steps steps per mode, "
                   "median; on = deterministic flag with torch's fill of uninitialised memory, on_nofill = without it"}
    line.update(gpu_identity(0))
    if args.dump_outputs and dumped is not None:
        import numpy as np
        out_dir = Path(args.dump_outputs)
        out_dir.mkdir(parents=True, exist_ok=True)
        for k, g in zip(GAUSS_KEYS, dumped):
            np.save(out_dir / f"grad_{k}.npy", g.detach().float().cpu().numpy())
    print(json.dumps(line))


if __name__ == "__main__":
    main()
