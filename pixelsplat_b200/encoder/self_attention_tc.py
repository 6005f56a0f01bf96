"""Host side of the wgmma self-attention kernel (csrc/self_attention_tc.cu): softmax(q k^T * scale) v
for ImageSelfAttention's ViT blocks, TF32 operands / FP32 accumulation on the tensor cores.

Reference semantics: /root/reference/src/model/transformer/attention.py:54-70 (z = None).  Forward AND
backward run on the tensor cores: the forward saves each row's (max, 1 / sum) so that the backward rebuilds
exactly the probabilities the forward used, TF32 roundings included, and differentiates the forward that
actually ran.

PIXELSPLAT_B200_SELF_ATTENTION=fp32 routes the module through torch's fp32 matmul/softmax instead
(for A/B precision checks); the default is the tensor-core kernel whenever the shape is the one it
is written for (256 tokens, 128-dim heads).
"""
from __future__ import annotations

import ctypes
import math
import os

import torch
from torch import Tensor

from .. import _lib

TOKENS, DIM_HEAD = 256, 128


def supported(x: Tensor, heads: int, dim_head: int, scale: float) -> bool:
    """Whether the kernel takes this call; a negative or non-finite scale is left to torch (the kernel takes the
    row max on unscaled logits, which only a scale >= 0 preserves)."""
    return (x.is_cuda and x.dtype == torch.float32 and x.dim() == 3 and x.shape[1] == TOKENS
            and dim_head == DIM_HEAD and 1 <= heads <= 16
            and 0.0 <= scale < math.inf
            and os.environ.get("PIXELSPLAT_B200_SELF_ATTENTION", "tf32") != "fp32")


def _launch(qkv: Tensor, heads: int, scale: float, debug_mode: int = 0) -> Tensor:
    n, L, three_inner = qkv.shape
    inner = three_inner // 3
    if debug_mode == 1:
        out = torch.empty((n, heads, L, L), dtype=torch.float32, device=qkv.device)
    else:
        out = torch.empty((n, L, inner), dtype=torch.float32, device=qkv.device)
    stream = torch.cuda.current_stream(qkv.device)
    rc = _lib.on_device(qkv.device, _lib.lib.ps_self_attention_forward, n, L, heads, inner // heads, ctypes.c_void_p(qkv.data_ptr()),
                                            ctypes.c_float(scale), ctypes.c_void_p(out.data_ptr()), debug_mode,
                                            ctypes.c_void_p(stream.cuda_stream))
    _lib.check(rc, "ps_self_attention_forward")
    return out


class _SelfAttentionTC(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv: Tensor, heads: int, scale: float):
        qkv = qkv.contiguous()
        n, L, three_inner = qkv.shape
        inner = three_inner // 3
        out = torch.empty((n, L, inner), dtype=torch.float32, device=qkv.device)
        stats = torch.empty((n, heads, L, 2), dtype=torch.float32, device=qkv.device)
        stream = torch.cuda.current_stream(qkv.device)
        rc = _lib.on_device(qkv.device, _lib.lib.ps_self_attention_forward_stats, n, L, heads, inner // heads,
                            ctypes.c_void_p(qkv.data_ptr()), ctypes.c_float(scale), ctypes.c_void_p(out.data_ptr()),
                            ctypes.c_void_p(stats.data_ptr()), ctypes.c_void_p(stream.cuda_stream))
        _lib.check(rc, "ps_self_attention_forward_stats")
        ctx.save_for_backward(qkv, out, stats)
        ctx.heads, ctx.scale = heads, scale
        return out

    @staticmethod
    def backward(ctx, dout: Tensor):
        qkv, out, stats = ctx.saved_tensors
        n, L, _ = qkv.shape
        H = ctx.heads
        dout = dout.contiguous().float()
        d_qkv = torch.empty_like(qkv)
        stream = torch.cuda.current_stream(qkv.device)
        rc = _lib.on_device(qkv.device, _lib.lib.ps_self_attention_backward, n, L, H, qkv.shape[-1] // (3 * H),
                            ctypes.c_void_p(qkv.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                            ctypes.c_void_p(dout.data_ptr()), ctypes.c_void_p(stats.data_ptr()),
                            ctypes.c_float(ctx.scale), ctypes.c_void_p(d_qkv.data_ptr()),
                            ctypes.c_void_p(stream.cuda_stream))
        _lib.check(rc, "ps_self_attention_backward")
        return d_qkv, None, None


def self_attention_tc(qkv: Tensor, heads: int, scale: float) -> Tensor:
    """qkv [n, 256, 3 * heads * 128] (to_qkv's output) -> [n, 256, heads * 128]."""
    return _SelfAttentionTC.apply(qkv, heads, scale)


def qk_logits_tc(qkv: Tensor, heads: int) -> Tensor:
    """Raw q k^T [n, heads, 256, 256] from the first tensor-core stage (tests only)."""
    return _launch(qkv.contiguous(), heads, 1.0, debug_mode=1)
