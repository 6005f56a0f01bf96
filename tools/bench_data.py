#!/usr/bin/env python
"""Times the data pipeline's per-view work on the host and the crop shim on the GPU:
  host       per view, one thread, host clock, over one seeded synthetic 360 x 640 JPEG (not a real RE10k frame):
             the reference's route restated (PIL decode + ToTensor, then rescale: float -> uint8 -> PIL
             Image.resize(LANCZOS) -> / 255, then the crop) against decode to uint8 only (what DatasetRE10k does);
  device     one re10k training batch, 7 scenes x (2 context + 4 target) = 42 views, 360 x 640 -> 256 x 256:
             csrc/image_resample.cu alone on device-resident views (rescale_and_crop_u8), and the whole device_shim
             from pinned host memory (the host-to-device copy included), CUDA events, median per call.
Prints one JSON line with the card and its power limit.  Nothing is written.

    python tools/bench_data.py [--steps 50] [--warmup 5] [--host-reps 20]
"""
import argparse
import io
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from pixelsplat_b200.data import crop_shim as cs  # noqa: E402
from tools.bench_depth import gpu_identity  # noqa: E402

SHAPE = (256, 256)
VIEWS = (7, 2, 4)   # scenes, context, target


def jpeg() -> bytes:
    rng = np.random.default_rng(0)
    yy, xx = np.meshgrid(np.linspace(0, 1, 360), np.linspace(0, 1, 640), indexing="ij")
    img = np.stack([0.5 + 0.3 * np.sin(7 * xx + c) * np.cos(5 * yy - c) for c in range(3)], -1) * 255
    img = np.clip(img + rng.normal(0, 12, img.shape), 0, 255).astype(np.uint8)
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, format="JPEG", quality=90)
    return buf.getvalue()


def host_times(data: bytes, reps: int) -> dict:
    torch.set_num_threads(1)                 # one loader worker is one thread

    def reference():
        x = torch.from_numpy(np.array(Image.open(io.BytesIO(data)))).permute(2, 0, 1).float() / 255   # ToTensor
        u = (x * 255).clip(min=0, max=255).type(torch.uint8).permute(1, 2, 0).numpy()
        r = np.array(Image.fromarray(u).resize((455, 256), Image.LANCZOS)) / 255
        return torch.tensor(r, dtype=torch.float32).permute(2, 0, 1)[:, :, 99:355]

    def decode_only():
        return np.array(Image.open(io.BytesIO(data)))

    out = {}
    for name, fn in (("reference_route", reference), ("decode_u8", decode_only)):
        fn()
        ts = []
        for _ in range(reps):
            t = time.perf_counter()
            fn()
            ts.append((time.perf_counter() - t) * 1e3)
        out[f"host_{name}_ms_per_view"] = statistics.median(ts)
    return out


def device_times(data: bytes, steps: int, warmup: int) -> dict:
    s, vc, vt = VIEWS
    view = torch.from_numpy(np.array(Image.open(io.BytesIO(data))))
    views = lambda v: view.expand(s, v, 360, 640, 3).contiguous().pin_memory()
    batch = {"context": {"image": views(vc), "intrinsics": torch.eye(3).expand(s, vc, 3, 3).contiguous()},
             "target": {"image": views(vt), "intrinsics": torch.eye(3).expand(s, vt, 3, 3).contiguous()},
             "flip": torch.arange(s) % 2 == 0}
    dev_images = view.expand(s * (vc + vt), 360, 640, 3).contiguous().cuda()
    dev_K = torch.eye(3, device="cuda").expand(s * (vc + vt), 3, 3)
    dev_flip = (torch.arange(s * (vc + vt), device="cuda") % 2).to(torch.uint8)
    runs = {"kernel": lambda: cs.rescale_and_crop_u8(dev_images, dev_K, SHAPE, dev_flip),
            "device_shim_from_pinned": lambda: cs.device_shim(batch, SHAPE)}
    out = {}
    for name, fn in runs.items():
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b))
        out[f"{name}_ms"] = statistics.median(ts)
    n = s * (vc + vt)
    out["kernel_us_per_view"] = out["kernel_ms"] * 1e3 / n
    out["views"] = n
    out["input_bytes"] = n * 360 * 640 * 3
    out["output_bytes"] = n * 3 * SHAPE[0] * SHAPE[1] * 4
    out["kernel_GBps"] = (out["input_bytes"] + out["output_bytes"]) / (out["kernel_ms"] * 1e-3) / 1e9
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_data: no CUDA device; the device times need an H100")
    data = jpeg()
    res = {"jpeg_bytes": len(data), **host_times(data, args.host_reps), **device_times(data, args.steps, args.warmup),
           **gpu_identity(0)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
