#!/usr/bin/env python
"""Times the PLY import of one re10k-sized scene: 393,216 Gaussians at SH degree 3 with normals (62 floats, 248 B
per record, a 97.5 MB file), exported by export_gaussians_ply from synthetic.scene_re10k_like into --output, then:
  kernel     ps_ply_unpack alone (csrc/ply_import.cu) into 16 coefficients, CUDA events over --steps launches, with
             the bytes it must move (248 B read, 244 B written per Gaussian) and the rate that gives;
  call       load_gaussians_ply end to end (host clock, ending in a device synchronise), median of --calls, and the
             same call split into its parts: the file read into the pinned buffer (host clock), the host-to-device
             copy and the kernel (CUDA events);
  host       the same unpack in numpy on the host (float32 arithmetic, then one copy of the result to the device),
             median of --calls.
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/bench_ply_import.py --output /tmp/ply_bench [--steps 200] [--calls 5]
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


def write_scene(path: Path) -> None:
    from pixelsplat_b200 import ply_export as pe, synthetic
    from pixelsplat_b200.decoder import Gaussians
    sc = synthetic.scene_re10k_like(seed=0, image_hw=(256, 256), context_views=2, gaussians_per_pixel=3, sh_degree=3)
    t = lambda x: x.to(DEV).contiguous()[None]
    pe.export_gaussians_ply(Gaussians(t(sc.means), t(sc.covariances), t(sc.harmonics), t(sc.opacities)),
                            torch.eye(4, device=DEV), path)


def events_ms(fn, steps: int) -> float:
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def numpy_route(path: Path):
    """The unpack on the host in float32 numpy (3DGS's own loader does this with plyfile), then one upload."""
    from pixelsplat_b200 import ply_import as pi
    data = path.read_bytes()
    layout = pi.parse_header(data)
    rec = np.frombuffer(data, "<f4", offset=layout.body_offset).reshape(layout.count, -1)
    col = {k: i for i, k in enumerate(layout.properties)}
    means = rec[:, [col["x"], col["y"], col["z"]]]
    q = rec[:, [col[f"rot_{i}"] for i in range(4)]]
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    w, x, y, z = q.T
    r = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                  np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                  np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)
    var = np.exp(2 * rec[:, [col[f"scale_{i}"] for i in range(3)]])
    cov = (r * var[:, None, :]) @ np.swapaxes(r, -1, -2)
    nc = 16
    harm = np.empty((layout.count, 3, nc), dtype=np.float32)
    for c in range(3):
        harm[:, c, 0] = rec[:, col[f"f_dc_{c}"]]
        harm[:, c, 1:] = rec[:, [col[f"f_rest_{c * 15 + k}"] for k in range(15)]]
    opac = 1 / (1 + np.exp(-rec[:, col["opacity"]]))
    out = [torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DEV) for a in (means, cov, harm, opac)]
    torch.cuda.synchronize()
    return out


def main() -> None:
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--output", type=Path, required=True, help="directory for the PLY file")
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--calls", type=int, default=5)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ply_import: no CUDA device; these numbers are only measured on the GPU")
    from pixelsplat_b200 import ply_import as pi
    path = args.output / "scene.ply"
    write_scene(path)
    n = 393_216

    layout, records = pi.read_ply_body(path, DEV)
    seen = []
    launch = pi._launch
    pi._launch = lambda *a: seen.append(a) or launch(*a)
    try:
        pi.unpack_records(records, layout.properties, layout.sh_degree)
    finally:
        pi._launch = launch
    (args_,) = seen
    kernel = lambda: launch(*args_)      # the ps_ply_unpack launch alone, without the host's descriptor set-up
    for _ in range(10):
        kernel()
    kernel_ms = events_ms(kernel, args.steps)
    moved = n * (248 + 244)

    calls, reads, copies, kernels = [], [], [], []
    for _ in range(args.calls + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pi.load_gaussians_ply(path, DEV)
        torch.cuda.synchronize()
        calls.append(time.perf_counter() - t0)
        # the same call in parts: the read (header and body into the pinned buffer), the copy, the kernel
        t0 = time.perf_counter()
        with open(path, "rb") as f:
            data_layout = pi.parse_header(f.read(1 << 20))
            f.seek(data_layout.body_offset)
            host = pi._pinned[0][:n * 62]
            f.readinto(memoryview(host.numpy()).cast("B"))
        reads.append(time.perf_counter() - t0)
        copies.append(events_ms(lambda: records.copy_(host.view(n, 62), non_blocking=True), 1) / 1e3)
        kernels.append(events_ms(kernel, 1) / 1e3)
    calls, reads, copies, kernels = calls[1:], reads[1:], copies[1:], kernels[1:]

    host = []
    for _ in range(args.calls):
        t0 = time.perf_counter()
        numpy_route(path)
        host.append(time.perf_counter() - t0)

    print(json.dumps({
        **gpu_identity(0), "gaussians": n, "file_bytes": path.stat().st_size,
        "kernel_ms": round(kernel_ms, 4), "kernel_bytes": moved, "kernel_gb_per_s": round(moved / kernel_ms / 1e6, 1),
        "call_ms_median": round(1e3 * statistics.median(calls), 2),
        "read_ms_median": round(1e3 * statistics.median(reads), 2),
        "copy_ms_median": round(1e3 * statistics.median(copies), 2),
        "kernel_in_call_ms_median": round(1e3 * statistics.median(kernels), 3),
        "numpy_host_ms_median": round(1e3 * statistics.median(host), 1),
        "calls": args.calls}))


if __name__ == "__main__":
    main()
