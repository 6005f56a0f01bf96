"""Cost of one test-time pose-alignment step on configs[1] (re10k-like 256x256, 2 context views x 3 Gaussians per
pixel = 393,216 Gaussians) with V = 1, 4 and 32 target views per call.

A step is what pixelsplat_b200.pose.align_poses runs: the fused-MSE forward of the twisted poses, the backward to the
[1, V, 6] twists and one Adam update.  It is timed with CUDA events (eager) in two forms, in alternating rounds
(median of each round, then the median and the spread over rounds):
  frozen   the Gaussians do not require grad: the camera-only rasterizer backward;
  gauss    the same step with the Gaussians requiring grad (their gradients are formed and dropped), which is what a
           frozen-Gaussian step cost before the camera-only backward existed.
torch.profiler gives the per-launch time of the backward kernels in a separate run.  Prints one JSON line, with the
card's name and power limit read in the same run.  Writes nothing.

    python tools/bench_pose_alignment.py [--rounds 6] [--iters 20] [--views 1,4,32]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import torch  # noqa: E402

from pixelsplat_b200 import synthetic  # noqa: E402
from pixelsplat_b200.pose import alignment_loss  # noqa: E402
from tools.bench_camera_grads import card  # noqa: E402

KERNELS = ("k_camera_bwd", "k_preprocess_bwd", "k_camera_finish", "k_composite_bwd2", "k_clear_pair_grads",
           "k_camera_setup_backward")


def setup(views: int):
    sc = synthetic.scene_re10k_like(seed=0, target_views=views)
    d = "cuda:0"
    t = lambda x: x.to(d)[None]
    ext, K, near, far = t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far)
    gauss = [t(sc.means), t(sc.covariances), t(sc.harmonics), t(sc.opacities)]
    bg = torch.zeros(1, views, 3, device=d)
    with torch.no_grad():
        target = torch.rand(1, views, 3, *sc.image_shape, device=d, generator=torch.Generator(d).manual_seed(0))
    xi = torch.full((1, views, 6), 1e-3, device=d, requires_grad=True)
    opt = torch.optim.Adam([xi], lr=1e-4)
    return dict(frozen=gauss, gauss=[g.clone().requires_grad_(True) for g in gauss], cams=(ext, K, near, far, bg),
                target=target, xi=xi, opt=opt)


def step(b, form: str):
    opt, xi = b["opt"], b["xi"]
    opt.zero_grad(set_to_none=True)
    for g in b["gauss"]:
        g.grad = None
    alignment_loss(xi, *b["cams"], *b[form], b["target"]).sum().backward()
    opt.step()


def timed(b, form: str) -> float:
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    step(b, form)
    e.record()
    e.synchronize()
    return a.elapsed_time(e)


def kernel_times(b) -> dict:
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for form in ("frozen", "gauss"):
        for _ in range(3):
            step(b, form)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                step(b, form)
            torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            name = next((k for k in KERNELS if k in ev.key), None)
            if name is None:
                continue
            dev_us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            per.setdefault(name, []).append({"kernel": ev.key[:120], "launches": ev.count,
                                             "us_per_launch": round(dev_us / max(ev.count, 1), 2)})
        out[form] = per
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--views", default="1,4,32")
    args = ap.parse_args()
    result = {"workload": "configs[1] re10k-like 256x256, 393216 Gaussians, eager pose-alignment step "
                          "(fused-MSE forward + backward + Adam)", "card": card(), "views": {}}
    for views in (int(v) for v in args.views.split(",")):
        b = setup(views)
        for _ in range(5):
            step(b, "frozen")
            step(b, "gauss")
        rounds = {"frozen": [], "gauss": []}
        for r in range(args.rounds):
            order = ("frozen", "gauss") if r % 2 == 0 else ("gauss", "frozen")
            for form in order:
                rounds[form].append(statistics.median(timed(b, form) for _ in range(args.iters)))
        entry = {f"step_ms_{form}": {"median": statistics.median(v), "min": min(v), "max": max(v)}
                 for form, v in rounds.items()}
        entry["speedup"] = entry["step_ms_gauss"]["median"] / entry["step_ms_frozen"]["median"]
        entry["kernels"] = kernel_times(b)
        result["views"][str(views)] = entry
        del b
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
