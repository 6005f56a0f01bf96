#!/usr/bin/env python
"""Times one refinement step of an exported re10k-sized scene: 393,216 Gaussians at SH degree 3 with normals (62
floats per record, pixelsplat_b200.ply_export.pack_viewer of synthetic.scene_re10k_like), refined against 2 context
views at 256 x 256 with 16 coefficients per channel:
  cuda    the step of ply_refine.refine_records (one RefineStep, its descriptor built once), split by CUDA events
          into the rasterizer forward + backward (render_views_mse and the backward of its loss) and the refinement
          call;
  kernel  ps_ply_refine_step alone: the prebuilt descriptor passed straight to the library, back to back under CUDA
          events, with the bytes it must move per Gaussian (computed from the shapes) and the rate that gives
          against 3.35 TB/s;
  torch   the same step built from torch ops: the unpack in torch float32 with autograd, the same rasterizer call and
          torch.optim.Adam with one group per property group, on SoA copies of the records.  This route is the one the
          GPU tests compare against (tests/test_ply_refine_gpu.py), and its unpack is tests/ply_refine_f64.py's
          unpack_torch, so the tool imports that test module; run it from the repository root.
The two routes run in alternating rounds of --steps steps each, after --warmup steps of each; medians over --rounds.
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/bench_ply_refine.py [--steps 50] [--warmup 10] [--rounds 5]
"""
import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tools.bench_depth import gpu_identity  # noqa: E402

DEV = "cuda:0"
FIELDS = ("means", "covariances", "harmonics", "opacities")


def scene():
    from pixelsplat_b200 import ply_export as pe, synthetic
    from pixelsplat_b200.decoder import Gaussians, render_views
    sc = synthetic.scene_re10k_like(seed=0, image_hw=(256, 256), context_views=2, gaussians_per_pixel=3, sh_degree=3,
                                 target_views=2)
    t = lambda x: x.to(DEV).contiguous()
    g = Gaussians(t(sc.means), t(sc.covariances), t(sc.harmonics), t(sc.opacities))
    ext, k = t(sc.extrinsics), t(sc.intrinsics)
    near, far = t(sc.near), t(sc.far)
    v = ext.shape[0]
    images = render_views(ext[None], k[None], near[None], far[None], (256, 256), torch.zeros(1, v, 3, device=DEV),
                          *(getattr(g, f)[None] for f in FIELDS))[0]
    records, names = pe.pack_viewer(g, ext[0])
    frame = pe.export_frame(g.means, ext[0])
    records[:, names.index("f_dc_0")] += 0.3    # a colour offset for the refinement to undo
    return records, names, frame, dict(extrinsics=ext, intrinsics=k, near=near, far=far, images=images)


class CudaRoute:
    def __init__(self, records, names, frame, views):
        from pixelsplat_b200 import ply_import as pi, ply_refine as pr
        from pixelsplat_b200.decoder import Gaussians
        self.names, self.frame, self.views = names, frame, views
        self.records = records.clone()
        self.m, self.v = torch.zeros_like(records), torch.zeros_like(records)
        n = records.shape[0]
        self.leaves = [torch.empty((1, n, 3), device=DEV), torch.empty((1, n, 3, 3), device=DEV),
                       torch.empty((1, n, 3, 16), device=DEV), torch.empty((1, n), device=DEV)]
        self.out = Gaussians(*(t[0] for t in self.leaves))
        pi.unpack_records(self.records, names, 3, frame=frame, out=self.out)
        for leaf in self.leaves:
            leaf.requires_grad_(True)
        self.t = 0
        self.step_fn = pr.RefineStep(names, 3, n, sh_coeffs=16, frame=frame)

    def step(self, marks=None):
        from pixelsplat_b200.decoder.cuda_splatting import render_views_mse
        w = self.views
        v = w["images"].shape[0]
        if marks:
            marks[0].record()
        sse, _, _ = render_views_mse(w["extrinsics"][None], w["intrinsics"][None], w["near"][None], w["far"][None],
                                     (256, 256), torch.zeros(1, v, 3, device=DEV), *self.leaves,
                                     target=w["images"][None], want_color=False)
        (sse.sum() / (v * 3 * 256 * 256)).backward()
        grads = [leaf.grad[0].contiguous() for leaf in self.leaves]
        for leaf in self.leaves:
            leaf.grad = None
        self.t += 1
        if marks:
            marks[1].record()
        self.step_fn(self.records, self.m, self.v, grads, self.out, self.t)
        if marks:
            marks[2].record()


class TorchRoute:
    def __init__(self, records, names, frame, views):
        from pixelsplat_b200 import ply_import as pi, ply_refine as pr, rasterizer
        from tests import ply_refine_f64 as rf
        self.rf, self.views = rf, views
        cols = rf.group_columns(names, 3)
        self.params = {k: records[:, c].clone().requires_grad_(True) for k, c in cols.items()}
        self.opt = torch.optim.Adam([{"params": [self.params[k]], "lr": pr.DEFAULT_LR[k]} for k in rf.GROUPS],
                                    lr=0.0, betas=pr.BETAS, eps=pr.EPS)
        self.blocks = [b.float().to(DEV) for b in pi.import_sh_blocks(frame.rotation, 3, rasterizer.get_sh_basis())]
        self.kw = dict(rotation=frame.rotation.float().to(DEV), center=frame.center, scale=float(frame.scale[0]))

    def step(self, marks=None):
        from pixelsplat_b200.decoder.cuda_splatting import render_views_mse
        w = self.views
        v = w["images"].shape[0]
        g = self.rf.unpack_torch(self.params, 3, 16, self.blocks, **self.kw)
        sse, _, _ = render_views_mse(w["extrinsics"][None], w["intrinsics"][None], w["near"][None], w["far"][None],
                                     (256, 256), torch.zeros(1, v, 3, device=DEV), *(g[f][None] for f in FIELDS),
                                     target=w["images"][None], want_color=False)
        self.opt.zero_grad(set_to_none=True)
        (sse.sum() / (v * 3 * 256 * 256)).backward()
        self.opt.step()


def timed(route, steps: int, split: bool):
    """(ms per step, raster ms per step, kernel ms per step); the split only for the CUDA route."""
    ev = lambda: torch.cuda.Event(enable_timing=True)
    start, end = ev(), ev()
    marks = [[ev(), ev(), ev()] for _ in range(steps)] if split else [None] * steps
    start.record()
    for mk in marks:
        route.step(mk)
    end.record()
    end.synchronize()
    total = start.elapsed_time(end) / steps
    if not split:
        return total, None, None
    return (total, sum(a.elapsed_time(b) for a, b, _ in marks) / steps,
            sum(b.elapsed_time(c) for _, b, c in marks) / steps)


def main() -> None:
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--warmup", type=int, default=10)
    p.add_argument("--rounds", type=int, default=5)
    args = p.parse_args()
    records, names, frame, views = scene()
    n, props = records.shape
    coeffs = 16
    gaussian = 4 * (3 + 9 + 3 * coeffs + 1)
    # read: record, exp_avg, exp_avg_sq and the four gradients; written: record, both moments and the Gaussian
    bytes_per = 2 * (3 * 4 * props + gaussian)
    cuda, torch_route = CudaRoute(records, names, frame, views), TorchRoute(records, names, frame, views)
    timed(cuda, args.warmup, False)
    timed(torch_route, args.warmup, False)
    rows = {"cuda": [], "raster": [], "kernel": [], "torch": []}
    for _ in range(args.rounds):
        total, raster, kernel = timed(cuda, args.steps, True)
        rows["cuda"].append(total)
        rows["raster"].append(raster)
        rows["kernel"].append(kernel)
        rows["torch"].append(timed(torch_route, args.steps, False)[0])
    med = {k: statistics.median(v) for k, v in rows.items()}
    # the kernel alone: the descriptor prebuilt (one call sets the pointers), then launched back to back
    import ctypes
    from pixelsplat_b200 import _lib
    grads = [torch.randn_like(t[0]) for t in cuda.leaves]
    cuda.step_fn(cuda.records, cuda.m, cuda.v, grads, cuda.out, cuda.t + 1)
    desc, stream = ctypes.byref(cuda.step_fn.desc), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    launch = lambda: _lib.check(_lib.lib.ps_ply_refine_step(desc, stream), "ps_ply_refine_step")
    for _ in range(args.warmup):
        launch()
    kernel_rounds = []
    for _ in range(args.rounds):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(4 * args.steps):
            launch()
        end.record()
        end.synchronize()
        kernel_rounds.append(start.elapsed_time(end) / (4 * args.steps))
    kernel_ms = statistics.median(kernel_rounds)
    tbs = bytes_per * n / (kernel_ms * 1e-3) / 1e12
    print(json.dumps({
        **gpu_identity(0), "gaussians": n, "properties": props, "views": int(views["images"].shape[0]),
        "image": [256, 256], "steps_per_round": args.steps, "rounds": args.rounds,
        "cuda_step_ms": med["cuda"], "cuda_raster_fwd_bwd_ms": med["raster"], "cuda_refine_call_ms": med["kernel"],
        "torch_step_ms": med["torch"], "cuda_step_rounds_ms": rows["cuda"], "torch_step_rounds_ms": rows["torch"],
        "kernel_back_to_back_ms": kernel_ms, "kernel_rounds_ms": kernel_rounds, "kernel_bytes_per_gaussian": bytes_per,
        "kernel_tb_per_s": tbs, "kernel_share_of_3_35_tb_per_s": tbs / 3.35}))


if __name__ == "__main__":
    main()
