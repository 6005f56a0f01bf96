#!/usr/bin/env python
"""Times the densification of an exported re10k-sized scene: 393,216 Gaussians at SH degree 3 with normals (62
floats per record, tools/bench_ply_refine.py's scene), 2 context views at 256 x 256:
  stats    ps_ply_densify_stats per launch, back to back under CUDA events, and its rate on the bytes it must move
           per Gaussian (V 16 B of d_means2d and radii read, 8 B read and 8 B written), against 3.35 TB/s;
  count / apply  ps_ply_densify_count (its two launches) and ps_ply_densify_apply, each back to back, at a seeded mix
           of about 10 % clone, 10 % split and 30 % prune; and the whole `densify_records` call with its one
           device-to-host read of the new count;
  step     one refinement step (render, backward, ps_ply_refine_step) with the statistics (a means2d leaf, its
           gradient from the backward and ps_ply_densify_stats) against one without, in alternating rounds: what the
           statistics cost a step.
Medians over --rounds.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/bench_ply_densify.py [--steps 50] [--warmup 10] [--rounds 5]
"""
import argparse
import ctypes
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tools.bench_depth import gpu_identity  # noqa: E402
from tools.bench_ply_refine import CudaRoute, scene  # noqa: E402

DEV = "cuda:0"


def per_launch(fn, launches: int, rounds: int) -> list[float]:
    out = []
    for _ in range(rounds):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(launches):
            fn()
        end.record()
        end.synchronize()
        out.append(start.elapsed_time(end) / launches)
    return out


class StatsRoute(CudaRoute):
    """CudaRoute's step with the densification statistics kept."""

    def __init__(self, *a):
        super().__init__(*a)
        n = self.records.shape[0]
        self.accum = torch.zeros(n, device=DEV)
        self.count = torch.zeros(n, dtype=torch.int32, device=DEV)

    def step(self, marks=None):
        from pixelsplat_b200 import ply_refine as pr
        from pixelsplat_b200.decoder.cuda_splatting import render_views_mse_means2d
        w = self.views
        v = w["images"].shape[0]
        means2d = torch.zeros((v, self.records.shape[0], 3), device=DEV, requires_grad=True)
        sse, _, _, radii = render_views_mse_means2d(
            w["extrinsics"][None], w["intrinsics"][None], w["near"][None], w["far"][None], (256, 256),
            torch.zeros(1, v, 3, device=DEV), *self.leaves, target=w["images"][None], means2d=means2d,
            want_color=False)
        (sse.sum() / (v * 3 * 256 * 256)).backward()
        pr.densify_stats(means2d.grad, radii, self.accum, self.count)
        grads = [leaf.grad[0].contiguous() for leaf in self.leaves]
        for leaf in self.leaves:
            leaf.grad = None
        self.t += 1
        self.step_fn(self.records, self.m, self.v, grads, self.out, self.t)


def timed_steps(route, steps: int) -> float:
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        route.step()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def mixed(records, names, g: torch.Generator):
    """Statistics and records for about 10 % clone, 10 % split, 30 % prune: per row, u < 0.1 selected and small,
    0.1 <= u < 0.2 selected and big, 0.2 <= u < 0.5 transparent, the rest kept."""
    import math
    n = records.shape[0]
    rec = records.clone()
    u = torch.rand(n, device=DEV, generator=g)
    scale = [names.index(f"scale_{k}") for k in range(3)]
    selected = u < 0.2
    rec[:, scale] = torch.where((u < 0.1)[:, None], math.log(0.005), rec[:, scale])
    rec[:, scale[0]] = torch.where(selected & (u >= 0.1), math.log(0.05), rec[:, scale[0]])
    rec[:, scale] = torch.where((~selected)[:, None], rec[:, scale].clamp(max=math.log(0.005)), rec[:, scale])
    o = names.index("opacity")
    rec[:, o] = torch.where((u >= 0.2) & (u < 0.5), -10.0, rec[:, o].abs())
    accum = torch.where(selected, 1e-3, 1e-5).float()
    count = torch.ones(n, dtype=torch.int32, device=DEV)
    return rec, accum, count


def main() -> None:
    from pixelsplat_b200 import _lib, ply_refine as pr
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--rounds", type=int, default=5)
    args = p.parse_args()
    records, names, frame, views = scene()
    n, props = records.shape
    v = int(views["images"].shape[0])
    g = torch.Generator(DEV).manual_seed(0)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    # statistics
    d2 = torch.randn((v, n, 3), device=DEV, generator=g) * 1e-4
    radii = torch.randint(-1, 4, (v, n), device=DEV, generator=g, dtype=torch.int32)
    accum, count = torch.zeros(n, device=DEV), torch.zeros(n, dtype=torch.int32, device=DEV)
    stats = lambda: _lib.lib.ps_ply_densify_stats(n, v, d2.data_ptr(), radii.data_ptr(), accum.data_ptr(),
                                                  count.data_ptr(), stream)
    for _ in range(args.warmup):
        stats()
    stats_ms = per_launch(stats, 4 * args.steps, args.rounds)
    stats_bytes = v * 16 + 16
    stats_tbs = stats_bytes * n / (statistics.median(stats_ms) * 1e-3) / 1e12

    # count and apply
    rec, acc, cnt = mixed(records, names, g)
    m, v2 = torch.randn_like(rec), torch.rand_like(rec)
    eps = torch.randn((2, n, 3), device=DEV, generator=g)
    cfg = pr.DensifyConfig()
    desc = pr.densify_desc(names, n, cfg, False)
    ws = torch.empty(pr.densify_workspace_bytes(n), dtype=torch.uint8, device=DEV)
    counts = torch.empty(4, dtype=torch.int64, device=DEV)
    count_fn = lambda: _lib.lib.ps_ply_densify_count(ctypes.byref(desc), rec.data_ptr(), acc.data_ptr(),
                                                     cnt.data_ptr(), ws.data_ptr(), ws.numel(), counts.data_ptr(),
                                                     stream)
    count_fn()
    kept, clones, splits, n_new = counts.tolist()
    outs = [torch.empty((n_new, props), device=DEV) for _ in range(3)]
    apply_fn = lambda: _lib.lib.ps_ply_densify_apply(ctypes.byref(desc), rec.data_ptr(), m.data_ptr(), v2.data_ptr(),
                                                     eps.data_ptr(), ws.data_ptr(), ws.numel(), counts.data_ptr(),
                                                     *(t.data_ptr() for t in outs), stream)
    for _ in range(args.warmup):
        count_fn()
        apply_fn()
    count_ms = per_launch(count_fn, 4 * args.steps, args.rounds)
    apply_ms = per_launch(apply_fn, 4 * args.steps, args.rounds)
    call = lambda: pr.densify_records(rec, m, v2, acc, cnt, names, cfg, prune_world=False, eps=eps, out=outs)
    call_ms = per_launch(call, args.steps, args.rounds)
    # apply: the records and moments of every input row read, the output rows written
    apply_bytes = 3 * 4 * props * (n + n_new) + n

    # refinement step with and without the statistics, alternating
    off, on = CudaRoute(records, names, frame, views), StatsRoute(records, names, frame, views)
    timed_steps(off, args.warmup)
    timed_steps(on, args.warmup)
    rows = {"off": [], "on": []}
    for _ in range(args.rounds):
        rows["off"].append(timed_steps(off, args.steps))
        rows["on"].append(timed_steps(on, args.steps))
    med = lambda xs: statistics.median(xs)
    print(json.dumps({
        **gpu_identity(0), "gaussians": n, "properties": props, "views": v, "image": [256, 256],
        "stats_ms": med(stats_ms), "stats_rounds_ms": stats_ms, "stats_bytes_per_gaussian": stats_bytes,
        "stats_tb_per_s": stats_tbs, "stats_share_of_3_35_tb_per_s": stats_tbs / 3.35,
        "mix": {"kept": kept, "clones": clones, "splits": splits, "n_new": n_new},
        "count_ms": med(count_ms), "apply_ms": med(apply_ms), "apply_bytes": apply_bytes,
        "apply_tb_per_s": apply_bytes / (med(apply_ms) * 1e-3) / 1e12, "densify_call_ms": med(call_ms),
        "step_off_ms": med(rows["off"]), "step_on_ms": med(rows["on"]), "step_off_rounds_ms": rows["off"],
        "step_on_rounds_ms": rows["on"]}))


if __name__ == "__main__":
    main()
