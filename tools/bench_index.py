"""Time the evaluation-index generator on one synthetic 300-frame scene at 256 x 256 (tests/index_util.py's
"rotate" family, whose walks end on overlap after ~80 frames), default configuration:

  kernel route     generate_scene_entry: one ps_view_overlap launch per context frame tried, one copy to the host,
                   the walk replayed there (host clock around the whole call, which ends in that copy)
  torch route      the reference's route restated in torch on the same GPU: two float32 project_rays
                   (near = far = None) per candidate and the host syncs of its comparisons (host clock)
  kernel alone     one launch over a full candidate range (273 frames, 2 directions), CUDA events over many launches

Bytes and operations are counted from the shapes; the card and its power limit are read in the same run.

    python tools/bench_index.py [--out RESULT.json]

The result is printed as one JSON line, and with --out also written to that file.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from pixelsplat_b200.evaluation import index_generator as ig  # noqa: E402
from tests import index_util  # noqa: E402

H = W = 256
# FP64 operations per ray of k_view_overlap, counted from csrc/epipolar_geometry.cu: the grid ray (~40), the move
# into the other camera (~30), four frame-line hits (~100) and the zero-depth and infinity projections (~50)
FLOPS_PER_RAY = 220


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def _rays(E, K):
    """World rays at the pixel centres of one camera (float32, as get_world_rays forms them)."""
    ys, xs = torch.meshgrid((torch.arange(H, device=E.device) + 0.5) / H, (torch.arange(W, device=E.device) + 0.5) / W,
                            indexing="ij")
    pix = torch.stack([xs.reshape(-1), ys.reshape(-1), torch.ones(H * W, device=E.device)], -1)
    d = pix @ torch.linalg.inv(K).T
    d = d / d.norm(dim=-1, keepdim=True)
    return E[:3, 3].expand(H * W, 3), d @ E[:3, :3].T


def _project(K, p):
    q = (p / (p[:, 2:] + torch.finfo(torch.float32).eps)).nan_to_num(posinf=1e8, neginf=-1e8)
    return q @ K[:2].T


def _in_bounds(xy):
    return ((xy >= -1e-6) & (xy <= 1 + 1e-6)).all(-1)


def torch_overlap(origins, dirs, E, K) -> torch.Tensor:
    """Share of the rays whose unbounded projection overlaps the image of camera (E, K): project_rays with
    near = far = None, restated in float32 torch."""
    w2c = torch.linalg.inv(E)
    o = origins @ w2c[:3, :3].T + w2c[:3, 3]
    d = dirs @ w2c[:3, :3].T
    ts, valids = [], []
    for dim, value in ((0, 0.0), (0, 1.0), (1, 0.0), (1, 1.0)):
        od = 1 - dim
        c = (value - K[dim, 2]) / K[dim, dim]
        t = (c * o[:, 2] - o[:, dim]) / (d[:, dim] - c * d[:, 2])
        other = K[od, 2] + K[od, od] * (o[:, od] * (c * d[:, 2] - d[:, dim]) + d[:, od] * (o[:, dim] - c * o[:, 2])) / (
            d[:, 2] * o[:, dim] - d[:, dim] * o[:, 2])
        xy = torch.stack([torch.full_like(other, value), other] if dim == 0 else [other, torch.full_like(other, value)], -1)
        z = o[:, 2] + t * d[:, 2]
        ts.append(t)
        valids.append(_in_bounds(xy) & (z > -1e-6) & (t > -1e-6))
    t, valid = torch.stack(ts), torch.stack(valids)
    lo_valid = valid.gather(0, torch.where(valid, t, torch.inf).min(0).indices[None])[0]
    hi_valid = valid.gather(0, torch.where(valid, t, -torch.inf).max(0).indices[None])[0]
    at_camera = o.norm(dim=-1) < 1e-6
    p = torch.where(at_camera[:, None], d, o)
    zero = _in_bounds(_project(K, p)) & (p[:, 2] > -1e-6) & ~((o[:, 2] < 1e-6) & ~at_camera)
    inf = _in_bounds(_project(K, d)) & (d[:, 2] > -1e-6)
    return ((zero | lo_valid) & (inf | hi_valid)).float().mean()


def torch_scene_entry(E, K, cfg, generator):
    """The reference's test_step on the GPU tensors: per candidate two projections and the 0-d tensor comparisons."""
    v = E.shape[0]
    for c in torch.randperm(v, generator=generator).tolist():
        co, cd = _rays(E[c], K[c])
        valid = []
        for step in (1, -1):
            k = c + step * cfg.min_distance
            while 0 <= k < v:
                ko, kd = _rays(E[k], K[k])
                overlap = min(torch_overlap(ko, kd, E[c], K[c]), torch_overlap(co, cd, E[k], K[k]))
                if cfg.min_overlap <= overlap <= cfg.max_overlap:
                    valid.append(k)
                if overlap < cfg.min_overlap or abs(k - c) > cfg.max_distance:
                    break
                k += step
        if valid:
            chosen = valid[int(torch.randint(0, len(valid), size=tuple(), generator=generator))]
            left, right = min(chosen, c), max(chosen, c)
            while True:
                targets = torch.randint(left, right + 1, (cfg.num_target_views,), generator=generator)
                if (targets.unique(return_counts=True)[1] == 1).all():
                    break
            return (left, right), tuple(sorted(targets.tolist()))
    return None


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", type=Path, default=None, help="also write the result to this JSON file")
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    E, K = (torch.from_numpy(a).to(dev) for a in index_util.trajectory("rotate"))
    cfg = ig.EvaluationIndexGeneratorCfg()
    result = {"card": card(), "scene": {"frames": E.shape[0], "h": H, "w": W, "family": "rotate"}}

    def kernel_route():
        return ig.generate_scene_entry(E, K, H, W, cfg, torch.Generator().manual_seed(cfg.seed))

    entry = kernel_route()                                   # warm-up (module load)
    times = []
    for _ in range(args.repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        kernel_route()
        times.append(time.perf_counter() - t0)
    result["kernel_route_s"] = {"min": min(times), "median": sorted(times)[len(times) // 2]}

    torch_entry = torch_scene_entry(E, K, cfg, torch.Generator().manual_seed(cfg.seed))   # warm-up
    times = []
    for _ in range(max(1, args.repeats // 2)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        torch_scene_entry(E, K, cfg, torch.Generator().manual_seed(cfg.seed))
        times.append(time.perf_counter() - t0)
    result["torch_route_s"] = {"min": min(times), "median": sorted(times)[len(times) // 2]}
    result["entries"] = {"kernel": [list(entry.context), list(entry.target)] if entry else None,
                         "torch": [list(x) for x in torch_entry] if torch_entry else None}

    first, count = ig.candidate_range(150, E.shape[0], cfg)
    for _ in range(10):
        ig.view_overlap_counts(E, K, H, W, 150, first, count)
    n = 200
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(n):
        ig.view_overlap_counts(E, K, H, W, 150, first, count)
    stop.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(stop) / n
    rays = 2 * count * H * W
    result["kernel_alone"] = {"candidates": count, "rays": rays, "ms": ms, "rays_per_s": rays / (ms * 1e-3),
                              "fp64_ops": rays * FLOPS_PER_RAY,
                              "fp64_tflops": rays * FLOPS_PER_RAY / (ms * 1e-3) / 1e12,
                              # each CTA reads its two cameras (16 + 9 floats each); the counts are 2 int32 a frame
                              "bytes": 2 * count * -(-H * W // 1024) * 2 * (16 + 9) * 4 + 8 * count}
    if args.out is not None:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(json.dumps(result, indent=1))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
