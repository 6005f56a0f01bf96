#!/usr/bin/env python
"""Times the PLY export of one re10k-sized scene (2 views x 256 x 256 x 3 Gaussians per pixel = 393,216 Gaussians,
SH degree 4, synthetic.scene_re10k_like) in both formats:
  kernel     ps_ply_pack alone (csrc/ply_export.cu), CUDA events over --steps launches, with the bytes it must move
             and the rate that gives;
  call       export_ply / export_gaussians_ply end to end: median, normalisation, the kernel, the device-to-host
             copy and the file write to --output (host clock, the file closed), median of --calls;
  host       a numpy restatement of the reference's host route on the same machine: the device-to-host copies, the
             quaternion composition on the host, then the structured array filled through list(map(tuple, ...)) and
             written with tofile (plyfile's binary write is one such call), for the reference's 17 floats and for
             the 62 of a full degree-3 record.
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/bench_ply_export.py --output /tmp/ply_bench [--steps 200] [--calls 5]
"""
import argparse
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tools.bench_depth import gpu_identity  # noqa: E402

DEV = "cuda:0"


def scene():
    from pixelsplat_b200 import synthetic
    from pixelsplat_b200.decoder import Gaussians
    sc = synthetic.scene_re10k_like(seed=0, image_hw=(256, 256), context_views=2, gaussians_per_pixel=3, sh_degree=4)
    n = sc.means.shape[0]
    g = torch.Generator().manual_seed(1)
    scales = (torch.randn(n, 3, generator=g) - 5).exp()
    rotations = torch.randn(n, 4, generator=g)
    ext = torch.eye(4)                                   # context view 0 yawed by 0.7 rad
    ext[:3, :3] = torch.tensor([[0.7648422, 0.0, 0.6442177], [0.0, 1.0, 0.0], [-0.6442177, 0.0, 0.7648422]])
    t = lambda x: x.to(DEV).contiguous()
    return (Gaussians(t(sc.means)[None], t(sc.covariances)[None], t(sc.harmonics)[None], t(sc.opacities)[None]),
            t(scales), t(rotations), t(ext))


def kernel_ms(call, steps: int, warmup: int) -> float:
    """Captures the ps_ply_pack launch `call` makes, then times that launch alone."""
    from pixelsplat_b200 import ply_export as pe
    seen = []
    pack = pe._pack
    pe._pack = lambda *a: seen.append(a) or pack(*a)
    try:
        call()
    finally:
        pe._pack = pack
    (args,) = seen
    for _ in range(warmup):
        pack(*args)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(steps):
        pack(*args)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def call_ms(call, calls: int) -> float:
    call()
    times = []
    for _ in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        call()
        times.append(1e3 * (time.perf_counter() - t0))
    return statistics.median(times)


def host_route_ms(gs, scales, rotations, ext, path: Path, rest: int, calls: int) -> float:
    """The reference's export_ply after its device-side median / quantile: everything it does on the host."""
    def route():
        means = gs.means[0]
        center = means.median(dim=0).values
        m = means - center
        s = m.abs().quantile(0.95, dim=0).max()
        c = np.float32(np.sqrt(0.5))
        frame = np.array([[c, c, 0], [-c, c, 0], [0, 0, 1]], np.float32) @ \
            np.array([[0, 0, 1], [-1, 0, 0], [0, -1, 0]], np.float32) @ np.linalg.inv(ext[:3, :3].cpu().numpy())
        pos = (m / s).cpu().numpy() @ frame.T
        q = rotations.cpu().numpy().astype(np.float64)
        x, y, z, w = (q / np.linalg.norm(q, axis=-1, keepdims=True)).T
        r = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], -1),
                      np.stack([2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)], -1),
                      np.stack([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], -1)], -2)
        a = frame.astype(np.float64) @ r
        qw = np.sqrt(np.maximum(1 + a[:, 0, 0] + a[:, 1, 1] + a[:, 2, 2], 1e-12)) / 2
        quat = np.stack([qw, (a[:, 2, 1] - a[:, 1, 2]) / (4 * qw), (a[:, 0, 2] - a[:, 2, 0]) / (4 * qw),
                         (a[:, 1, 0] - a[:, 0, 1]) / (4 * qw)], -1)
        harmonics = gs.harmonics[0][..., :(1 + rest // 3)].cpu().numpy()
        attrs = np.concatenate([pos, np.zeros_like(pos), harmonics[..., 0], harmonics[..., 1:].reshape(len(pos), -1),
                                gs.opacities[0][:, None].cpu().numpy(), (scales / s).log().cpu().numpy(), quat], axis=1)
        names = [f"p{i}" for i in range(attrs.shape[1])]
        elements = np.empty(len(pos), dtype=[(k, "f4") for k in names])
        elements[:] = list(map(tuple, attrs))
        elements.tofile(path)
    return call_ms(route, calls)


def main() -> None:
    p = argparse.ArgumentParser()
    p.add_argument("--output", type=Path, required=True, help="directory the timed files are written to")
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--calls", type=int, default=5)
    p.add_argument("--host-calls", type=int, default=3)
    args = p.parse_args()
    from pixelsplat_b200 import ply_export as pe
    args.output.mkdir(parents=True, exist_ok=True)
    gs, scales, rotations, ext = scene()
    n = gs.means.shape[1]
    one = lambda t: t[0]
    ref = lambda: pe.export_ply(ext, one(gs.means), scales, rotations, one(gs.harmonics), one(gs.opacities),
                                args.output / "reference.ply")
    viewer = lambda: pe.export_gaussians_ply(gs, ext, args.output / "viewer.ply")
    # bytes the kernel must move: inputs it reads (harmonics: the coefficients it uses; the rest in full), output
    read_ref = n * 4 * (3 + 3 + 4 + 3 + 1)
    read_viewer = n * 4 * (3 + 9 + 3 * 16 + 1)
    out = {"gaussians": n, **gpu_identity(0)}
    for name, call, floats, read in (("reference", ref, 17, read_ref), ("viewer", viewer, 62, read_viewer)):
        k = kernel_ms(call, args.steps, args.warmup)
        moved = read + n * 4 * floats
        out[name] = {"kernel_ms": round(k, 4), "kernel_bytes": moved, "kernel_gb_s": round(moved / k / 1e6, 1),
                     "call_ms": round(call_ms(call, args.calls), 2), "file_bytes": (args.output / f"{name}.ply").stat().st_size}
    out["host_route_ms"] = {"dc_only_17": round(host_route_ms(gs, scales, rotations, ext, args.output / "host17.bin", 0,
                                                              args.host_calls), 1),
                            "degree3_62": round(host_route_ms(gs, scales, rotations, ext, args.output / "host62.bin", 45,
                                                              args.host_calls), 1)}
    for f in args.output.iterdir():
        f.unlink()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
