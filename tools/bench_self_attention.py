#!/usr/bin/env python
"""Times the wgmma self-attention kernel (csrc/self_attention_tc.cu) against torch's own paths for
the same contraction -- fp32 matmul + softmax (what the reference runs, attention.py:54-70), the
same with TF32 matmuls allowed, and F.scaled_dot_product_attention -- at ImageSelfAttention's shape
(256 tokens, 4 heads x 128) for a range of image counts.  CUDA events, L2 not flushed (the whole
working set is a few MB; it is L2-resident in the real step too, straight out of the to_qkv GEMM).

    python tools/bench_self_attention.py            # prints one JSON line
"""
import json
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def timed(fn, iters=50, warmup=10):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3          # microseconds


def main():
    from pixelsplat_b200.encoder import self_attention_tc as sa
    dev = torch.device("cuda", 0)
    heads, L, d = 4, 256, 128
    scale = d ** -0.5
    rows = []
    for n in (2, 14, 37, 132):
        qkv = torch.randn(n, L, 3 * heads * d, device=dev)

        def explicit():
            q, k, v = (t.reshape(n, L, heads, d).transpose(1, 2) for t in qkv.chunk(3, dim=-1))
            p = torch.softmax(torch.matmul(q, k.transpose(-1, -2)) * scale, dim=-1)
            return torch.matmul(p, v).transpose(1, 2).reshape(n, L, heads * d)

        def sdpa():
            q, k, v = (t.reshape(n, L, heads, d).transpose(1, 2) for t in qkv.chunk(3, dim=-1))
            return F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(n, L, heads * d)

        t_tc = timed(lambda: sa.self_attention_tc(qkv, heads, scale))
        torch.backends.cuda.matmul.allow_tf32 = False
        t_fp32 = timed(explicit)
        torch.backends.cuda.matmul.allow_tf32 = True
        t_tf32 = timed(explicit)
        torch.backends.cuda.matmul.allow_tf32 = False
        t_sdpa = timed(sdpa)
        # forward + backward on the wgmma pair
        qg = qkv.clone().requires_grad_(True)
        wgt = torch.randn(n, L, heads * d, device=dev)

        def fb():
            qg.grad = None
            (sa.self_attention_tc(qg, heads, scale) * wgt).sum().backward()

        t_fb_tc = timed(fb, iters=30, warmup=5)
        ref = explicit().double()
        err = float((sa.self_attention_tc(qkv, heads, scale).double() - ref).abs().max() / ref.abs().max())
        flops = n * heads * 2 * (2.0 * L * L * d)
        rows.append({"images": n, "ctas": 2 * heads * n, "wgmma_us": t_tc, "torch_fp32_us": t_fp32,
                     "torch_tf32_us": t_tf32, "torch_sdpa_us": t_sdpa,
                     "fwd_bwd_wgmma_us": t_fb_tc, "wgmma_tflops": flops / t_tc * 1e-6,
                     "rel_err_vs_torch_fp32": err})
    print(json.dumps({"what": "self-attention 256 tokens x 4 heads x 128; forward, and forward + backward (incl. the loss ops)", "rows": rows}))


if __name__ == "__main__":
    main()
