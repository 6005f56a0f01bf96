"""Per-launch times of the SH forward and the preprocess backward on configs[1] (re10k-like 256x256, 2 context views x 3
Gaussians per pixel = 393,216 Gaussians, SH degree 4), and the cost of a forward-only render.

  --mode kernels   bench.py's step (forward + backward through render_views, captured once into a CUDA graph) with V
                   target views per call, replayed --replays times under torch.profiler: microseconds per launch of
                   every rasterizer kernel.
  --mode forward   a no-grad render_views of the same scene, V = 1, timed with CUDA events: --rounds rounds of --iters
                   calls, the median per round, then the median and the range over rounds.

Prints one JSON line, with the card's name and power limit read in the same run.  Writes nothing.

    python tools/bench_preprocess_bwd.py --mode kernels [--views 1,4] [--replays 400]
    python tools/bench_preprocess_bwd.py --mode forward [--rounds 5] [--iters 200]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

import bench  # noqa: E402
from tools.bench_camera_grads import card  # noqa: E402

KERNELS = ("k_preprocess_bwd", "k_sh_color", "k_preprocess", "k_camera_bwd", "k_composite_bwd2", "k_composite_fwd2",
           "k_tile_sort", "k_scatter", "k_clear_pair_grads")


def scene(views: int) -> dict:
    d = {k: v.cuda() for k, v in bench.scene_host_tensors(bench.make_scene(0, views), pin=False).items()}
    for k in bench.GAUSS_KEYS:
        d[k].requires_grad_(True)
    return d


def kernel_times(views: int, replays: int) -> dict:
    from torch.profiler import ProfilerActivity, profile

    from pixelsplat_b200 import rasterizer
    d = scene(views)
    d_img = torch.randn((1, views, 3, *bench.IMAGE), generator=torch.Generator().manual_seed(7)).cuda()
    rasterizer.set_capacity_check("sync")
    bench.render_step(d, d_img, views)
    rasterizer.set_capacity_check("deferred")
    graph, _, states = bench.capture_step(d, d_img, views)
    for _ in range(20):
        graph.replay()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(replays):
            graph.replay()
        torch.cuda.synchronize()
    for st in states:
        st.verify()
    per = {}
    for ev in prof.key_averages():
        name = next((k for k in KERNELS if k in ev.key and (k != "k_preprocess" or "k_preprocess_bwd" not in ev.key)),
                    None)
        if name is None:
            continue
        dev_us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        per[ev.key[:100]] = {"launches": ev.count, "us_per_launch": round(dev_us / max(ev.count, 1), 2)}
    return per


def forward_times(rounds: int, iters: int) -> dict:
    from pixelsplat_b200.decoder import render_views
    d = scene(1)
    bg = torch.zeros((1, 1, 3), device="cuda")
    args = (d["extrinsics"][None], d["intrinsics"][None], d["near"][None], d["far"][None], bench.IMAGE, bg,
            *[d[k].detach() for k in bench.GAUSS_KEYS])
    with torch.no_grad():
        for _ in range(20):
            render_views(*args)
        med = []
        for _ in range(rounds):
            ts = []
            for _ in range(iters):
                a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                render_views(*args)
                e.record()
                e.synchronize()
                ts.append(a.elapsed_time(e))
            med.append(statistics.median(ts))
    return {"ms_per_render": round(statistics.median(med), 4), "round_medians": [round(m, 4) for m in med]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", choices=["kernels", "forward"], required=True)
    ap.add_argument("--views", default="1,4")
    ap.add_argument("--replays", type=int, default=400)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    out = {"card": card(), "mode": args.mode}
    if args.mode == "kernels":
        out["replays"] = args.replays
        out["views"] = {v: kernel_times(int(v), args.replays) for v in args.views.split(",")}
    else:
        out.update(forward_times(args.rounds, args.iters))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
