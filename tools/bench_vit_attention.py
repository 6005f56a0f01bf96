"""Times the ViT attention kernel (csrc/vit_attention.cu) against DINO's explicit fp32 attention and against
torch's F.scaled_dot_product_attention in fp32, at the re10k training shape: 14 images x 1025 tokens x 12 heads x 64
(dino_vitb8 at 256 x 256).  Forward and forward+backward, device-timed with CUDA events, the three routes
alternating round by round; reports the median per route and the peak memory one call allocates.

    python tools/bench_vit_attention.py [--n 14] [--tokens 1025] [--heads 12] [--rounds 7] [--iters 10]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from pixelsplat_b200.encoder.vit_attention import vit_attention  # noqa: E402


def explicit(qkv, H, scale):
    B, N, C3 = qkv.shape
    q, k, v = qkv.reshape(B, N, 3, H, C3 // (3 * H)).permute(2, 0, 3, 1, 4)
    attn = ((q @ k.transpose(-2, -1)) * scale).softmax(dim=-1)
    return (attn @ v).transpose(1, 2).reshape(B, N, C3 // 3)


def sdpa(qkv, H, scale):
    B, N, C3 = qkv.shape
    q, k, v = qkv.reshape(B, N, 3, H, C3 // (3 * H)).permute(2, 0, 3, 1, 4)
    return F.scaled_dot_product_attention(q, k, v, scale=scale).transpose(1, 2).reshape(B, N, C3 // 3)


ROUTES = {"kernel": lambda x, H, s: vit_attention(x, H, s), "dino_explicit_fp32": explicit, "sdpa_fp32": sdpa}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=14)
    ap.add_argument("--tokens", type=int, default=1025)
    ap.add_argument("--heads", type=int, default=12)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = "cuda:0"
    scale = 64 ** -0.5
    qkv = torch.randn(a.n, a.tokens, 3 * a.heads * 64, device=dev)
    dout = torch.randn(a.n, a.tokens, a.heads * 64, device=dev)
    x = qkv.clone().requires_grad_(True)

    def step(route, bwd):
        if bwd:
            ROUTES[route](x, a.heads, scale).backward(dout)
            x.grad = None
        else:
            with torch.no_grad():
                ROUTES[route](qkv, a.heads, scale)

    times = {(r, b): [] for r in ROUTES for b in (False, True)}
    peak = {}
    for r in ROUTES:
        for b in (False, True):
            step(r, b)                                                   # warm-up
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            step(r, b)
            torch.cuda.synchronize()
            peak[(r, b)] = torch.cuda.max_memory_allocated() - base
    for _ in range(a.rounds):
        for r in ROUTES:
            for b in (False, True):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    step(r, b)
                e1.record()
                e1.synchronize()
                times[(r, b)].append(e0.elapsed_time(e1) / a.iters)
    res = {f"{r}_{'fwd_bwd' if b else 'fwd'}": {"ms": round(statistics.median(t), 3),
                                                "peak_mb": round(peak[(r, b)] / 2 ** 20, 1)}
           for (r, b), t in times.items()}
    print(json.dumps({"shape": [a.n, a.tokens, a.heads * 64], "gpu": torch.cuda.get_device_name(), **res}))


if __name__ == "__main__":
    main()
