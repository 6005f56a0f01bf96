#!/usr/bin/env python
"""Counts, on the CPU, how much of the tile lists the compositor's per-block cull finds dead: the numbers behind the
per-tile live lists (ps_common.cuh, kLivePosLimit).

For one target view of the bench scene (synthetic.scene_re10k_like with bench.py's parameters), oracle/raster_torch.py's
preprocess and tile binning give the depth-sorted per-tile lists; each entry gets the alpha >= 1/255 box that
k_preprocess writes as its cull record (half-extents sqrt(2 ln(255 o) Sigma_ii) * 1.001 + 0.01, here from the inverse
of the conic), and is tested against its tile's 16x16 rectangle and the tile's eight 8x4 blocks with the compositor's
test.  Prints the instance count, the mean and longest list, the share of entries whose box misses their whole tile,
the share with opacity < 1/255, the (entry, block) hits over the 8 N the per-block cull used to test, and opacity
quantiles of the visible Gaussians.  Nothing is written.

    python tools/count_live_entries.py [--seed 0] [--image 256]
"""
import argparse
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from oracle import raster_torch as rt  # noqa: E402
from pixelsplat_b200 import synthetic  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=0, help="scene seed (bench.py's pool uses 0, 1, 2, 3)")
    ap.add_argument("--image", type=int, default=256)
    args = ap.parse_args()
    W = H = args.image
    sc = synthetic.scene_re10k_like(seed=args.seed, image_hw=(H, W), context_views=2, gaussians_per_pixel=3,
                                    sh_degree=4, target_views=1)
    a = rt.prepare_view(sc.means, sc.covariances, sc.harmonics, sc.opacities, sc.extrinsics[0], sc.intrinsics[0],
                        sc.near[0], sc.far[0])
    with torch.no_grad():
        pre = rt.preprocess(a["means"], a["cov6"], a["opac"], None, torch.zeros(a["means"].shape[0], 3), a["vm"],
                            a["pm"], a["campos"], a["tanfovx"], a["tanfovy"], W, H, 0)
        keys, values, ranges = rt.bin_tiles(pre, W, H)
        n = values.numel()
        gx = (W + 15) // 16
        tile = keys >> 32
        tx, ty = (tile % gx).float(), (tile // gx).float()
        op = pre["opacity"][values]
        A, B, C = pre["conic"][values].unbind(-1)
        det = A * C - B * B
        tau2 = 2 * (torch.log(torch.clamp(op * 255, min=1.0)) + 0.01)
        ex = torch.sqrt(tau2 * C / det) * 1.001 + 0.01       # covariance diagonal = (C, A) / det of the conic
        ey = torch.sqrt(tau2 * A / det) * 1.001 + 0.01
        never = op * 255 < 1 - 1e-3
        x, y = pre["xy"][values].unbind(-1)

        def meets(x0, x1, y0, y1):
            return (~never) & (x + ex >= x0) & (x - ex <= x1) & (y + ey >= y0) & (y - ey <= y1)

        live = meets(tx * 16, tx * 16 + 15, ty * 16, ty * 16 + 15)
        hits = sum(int(meets(tx * 16 + (b & 1) * 8, tx * 16 + (b & 1) * 8 + 7,
                             ty * 16 + (b >> 1) * 4, ty * 16 + (b >> 1) * 4 + 3).sum()) for b in range(8))
        cnt = (ranges[:, 1] - ranges[:, 0]).float()
        q = torch.quantile(pre["opacity"][pre["visible"]], torch.tensor([0.1, 0.5, 0.9]))
    print(f"seed {args.seed}, {W}x{H}: instances N = {n}, mean per tile {float(cnt.mean()):.0f}, "
          f"longest tile {int(cnt.max())}")
    print(f"entries whose box misses their whole tile: {100 * (1 - float(live.float().mean())):.1f} % "
          f"(opacity < 1/255: {100 * float(never.float().mean()):.1f} %)")
    print(f"(entry, block) hits: {100 * hits / (8 * n):.1f} % of 8 N, "
          f"{100 * hits / (8 * int(live.sum())):.1f} % of 8 x the tile-live entries")
    print("visible opacity 10/50/90 % quantiles: " + " / ".join(f"{v:.3f}" for v in q.tolist()))


if __name__ == "__main__":
    main()
