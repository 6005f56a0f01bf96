"""Cost of camera gradients in the rasterizer backward, on configs[1] (re10k-like 256x256, 2 context views x 3
Gaussians per pixel = 393,216 Gaussians) at 1 and 4 target views per call.

Eager forward + backward through render_views with the Gaussians requiring grad; the backward is timed with CUDA
events, with and without extrinsics requiring grad, in alternating rounds (median of each round, then the median and
the spread over rounds).  torch.profiler gives the per-launch time of the camera-gradient instantiation of
k_preprocess_bwd, its default instantiation and the finish kernel.  Prints one JSON line, with the card's name and
power limit read in the same run.  Writes nothing.

    python tools/bench_camera_grads.py [--rounds 6] [--iters 20]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

from pixelsplat_b200 import synthetic  # noqa: E402
from pixelsplat_b200.decoder.cuda_splatting import render_views  # noqa: E402


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        info["power_limit_w"] = float(out.stdout.strip().splitlines()[0])
    except Exception as e:       # the number is then reported as unknown, not guessed
        info["power_limit_error"] = str(e)
    return info


def setup(views: int):
    sc = synthetic.scene_re10k_like(seed=0, target_views=views)
    d = "cuda:0"
    t = lambda x: x.to(d)[None]
    g = [t(sc.means).requires_grad_(True), t(sc.covariances).requires_grad_(True),
         t(sc.harmonics).requires_grad_(True), t(sc.opacities).requires_grad_(True)]
    return (t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far), sc.image_shape,
            torch.zeros(1, views, 3, device=d), g)


def step(cams, cam_grad: bool, timed: bool):
    ext, K, near, far, hw, bg, g = cams
    for x in g:
        x.grad = None
    e = ext.clone().requires_grad_(cam_grad)
    img = render_views(e, K, near, far, hw, bg, *g)
    loss = img.square().mean()
    if not timed:
        loss.backward()
        return None
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    loss.backward()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def kernel_times(cams) -> dict:
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        step(cams, True, False)
        step(cams, False, False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            step(cams, True, False)
            step(cams, False, False)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        name = ev.key
        if "k_preprocess_bwd" in name or "k_camera_finish" in name or "k_camera_setup_backward" in name:
            key = ("k_camera_finish" if "k_camera_finish" in name else
                   "k_camera_setup_backward" if "k_camera_setup_backward" in name else
                   "k_preprocess_bwd<CAM>" if name.rstrip().endswith("true>") or "Lb1EE" in name or ", true>" in name
                   else "k_preprocess_bwd")
            dev_us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            out.setdefault(key, []).append({"kernel": name, "launches": ev.count, "us_per_launch": dev_us / max(ev.count, 1)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    result = {"workload": "configs[1] re10k-like 256x256, 393216 Gaussians, eager render_views backward",
              "card": card(), "views": {}}
    for views in (1, 4):
        cams = setup(views)
        for _ in range(5):
            step(cams, False, False)
            step(cams, True, False)
        rounds = {False: [], True: []}
        for r in range(args.rounds):
            order = (False, True) if r % 2 == 0 else (True, False)
            for cg in order:
                rounds[cg].append(statistics.median(step(cams, cg, True) for _ in range(args.iters)))
        entry = {}
        for cg, name in ((False, "backward_ms_without_camera_grads"), (True, "backward_ms_with_camera_grads")):
            entry[name] = {"median": statistics.median(rounds[cg]), "min": min(rounds[cg]), "max": max(rounds[cg])}
        entry["kernels"] = kernel_times(cams)
        result["views"][str(views)] = entry
        del cams
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
