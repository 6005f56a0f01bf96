#!/usr/bin/env python
"""Times 3DGS's L1 + D-SSIM loss (csrc/l1_dssim.cu, pixelsplat_b200.loss.l1_dssim) and the refinement step that uses it:
  kernel     ps_l1_dssim with the gradient, launched back to back under CUDA events at [2, 3, 256, 256],
             [4, 3, 256, 256] and [1, 3, 360, 640], with its rate on the bytes it must move (p and g read, d_p written:
             12 bytes a pixel and channel) against 3.35 TB/s;
  torch      the same loss and gradient from torch ops: 3DGS's conv2d(padding=5, groups=C) SSIM and the mean absolute
             difference, forward + backward through autograd (float32, TF32 off), at the same shapes;
  refine     one refinement step of bench_ply_refine.py's scene (393,216 Gaussians at SH degree 3, 2 views at
             256 x 256): the fused-MSE step and the L1 + D-SSIM step (colour render, loss, rasterizer backward,
             ps_ply_refine_step), in alternating rounds after a warm-up of each.
Medians over --rounds.  Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/bench_l1_dssim.py [--steps 50] [--warmup 10] [--rounds 5]
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
from tools.bench_ply_refine import DEV, CudaRoute, scene, timed  # noqa: E402

SHAPES = [(2, 3, 256, 256), (4, 3, 256, 256), (1, 3, 360, 640)]


def events_ms(fn, count: int, rounds: int) -> list[float]:
    out = []
    for _ in range(rounds):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(count):
            fn()
        end.record()
        end.synchronize()
        out.append(start.elapsed_time(end) / count)
    return out


def kernel_and_torch(shape, steps: int, warmup: int, rounds: int) -> dict:
    from pixelsplat_b200 import _lib
    from tests import l1_dssim_f64 as lf
    n, c, h, w = shape
    g = torch.Generator(DEV).manual_seed(0)
    p, t = torch.rand(shape, device=DEV, generator=g), torch.rand(shape, device=DEV, generator=g)
    size = ctypes.c_size_t()
    _lib.check(_lib.lib.ps_l1_dssim_workspace_bytes(n, c, h, w, ctypes.byref(size)), "ps_l1_dssim_workspace_bytes")
    ws = torch.empty(size.value, dtype=torch.uint8, device=DEV)
    out, d_p = torch.empty(n, device=DEV), torch.empty_like(p)
    stream = torch.cuda.current_stream().cuda_stream
    args = (n, c, h, w, p.data_ptr(), t.data_ptr(), 0.2, out.data_ptr(), None, None, d_p.data_ptr(), ws.data_ptr(),
            ws.numel(), stream)
    launch = lambda: _lib.check(_lib.lib.ps_l1_dssim(*args), "ps_l1_dssim")
    pg = p.clone().requires_grad_(True)

    def torch_route():
        pg.grad = None
        lf.loss_3dgs_torch(pg, t, 0.2).sum().backward()

    events_ms(launch, warmup, 1)
    events_ms(torch_route, warmup, 1)
    kernel, torch_rows = [], []
    for _ in range(rounds):
        kernel += events_ms(launch, 4 * steps, 1)
        torch_rows += events_ms(torch_route, steps, 1)
    k = statistics.median(kernel)
    moved = 12 * n * c * h * w
    return {"shape": list(shape), "kernel_ms": k, "kernel_rounds_ms": kernel, "kernel_bytes": moved,
            "kernel_tb_per_s": moved / (k * 1e-3) / 1e12, "kernel_share_of_3_35_tb_per_s": moved / (k * 1e-3) / 3.35e12,
            "torch_ms": statistics.median(torch_rows), "torch_rounds_ms": torch_rows}


class DssimRoute(CudaRoute):
    """CudaRoute's step with ply_refine's L1 + D-SSIM objective: the colour render, the loss summed over the views,
    the rasterizer backward, then the same RefineStep."""

    def step(self, marks=None):
        from pixelsplat_b200.decoder import render_views
        from pixelsplat_b200.loss import l1_dssim
        w = self.views
        v = w["images"].shape[0]
        if marks:
            marks[0].record()
        color = render_views(w["extrinsics"][None], w["intrinsics"][None], w["near"][None], w["far"][None],
                             (256, 256), torch.zeros(1, v, 3, device=DEV), *self.leaves)
        l1_dssim(color[0], w["images"]).sum().backward()
        grads = [leaf.grad[0].contiguous() for leaf in self.leaves]
        for leaf in self.leaves:
            leaf.grad = None
        self.t += 1
        if marks:
            marks[1].record()
        self.step_fn(self.records, self.m, self.v, grads, self.out, self.t)
        if marks:
            marks[2].record()


def main() -> None:
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--rounds", type=int, default=5)
    args = p.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    losses = [kernel_and_torch(s, args.steps, args.warmup, args.rounds) for s in SHAPES]
    records, names, frame, views = scene()
    routes = {"mse": CudaRoute(records, names, frame, views), "l1_dssim": DssimRoute(records, names, frame, views)}
    for r in routes.values():
        timed(r, args.warmup, False)
    rows = {k: [] for k in routes}
    for _ in range(args.rounds):
        for k, r in routes.items():
            rows[k].append(timed(r, args.steps, False)[0])
    print(json.dumps({
        **gpu_identity(0), "loss": losses, "refine_gaussians": int(records.shape[0]), "refine_views": 2,
        "refine_image": [256, 256], "steps_per_round": args.steps, "rounds": args.rounds,
        "refine_mse_step_ms": statistics.median(rows["mse"]),
        "refine_l1_dssim_step_ms": statistics.median(rows["l1_dssim"]),
        "refine_mse_rounds_ms": rows["mse"], "refine_l1_dssim_rounds_ms": rows["l1_dssim"]}))


if __name__ == "__main__":
    main()
