"""Host side of the flash-style ViT attention kernel (csrc/vit_attention.cu): softmax(q k^T * scale) v for DINO's
ViT blocks, TF32 operands / FP32 accumulation on the tensor cores, any token count, 64-dim heads.

The forward saves the per-row log-sum-exp; the backward recomputes the probabilities from it (FlashAttention-2),
so no [L, L] tensor is ever stored, and it uses no float atomics, so repeated backward runs give the same bits.

PIXELSPLAT_B200_VIT_ATTENTION=fp32 routes DINO's Attention through its explicit torch formula instead (for A/B
precision checks); the default is the kernel whenever the input is CUDA fp32 with 64-dim heads.
"""
from __future__ import annotations

import ctypes
import os

import torch
from torch import Tensor

from .. import _lib

DIM_HEAD, MAX_TOKENS, MAX_HEADS = 64, 16384, 16


def supported(x: Tensor, heads: int, dim_head: int) -> bool:
    return (x.is_cuda and x.dtype == torch.float32 and dim_head == DIM_HEAD and 1 <= heads <= MAX_HEADS
            and 1 <= x.shape[1] <= MAX_TOKENS
            and os.environ.get("PIXELSPLAT_B200_VIT_ATTENTION", "tf32") != "fp32")


def workspace_bytes(n: int, tokens: int, heads: int, dim_head: int = DIM_HEAD) -> int:
    out = ctypes.c_size_t()
    _lib.check(_lib.lib.ps_vit_attention_backward_workspace_bytes(n, tokens, heads, dim_head, ctypes.byref(out)),
               "ps_vit_attention_backward_workspace_bytes")
    return out.value


def forward(qkv: Tensor, heads: int, scale: float) -> tuple[Tensor, Tensor]:
    """qkv [n, L, 3 * heads * 64] (contiguous) -> (out [n, L, heads * 64], lse [n, heads, L])."""
    n, L, three_inner = qkv.shape
    inner = three_inner // 3
    out = torch.empty((n, L, inner), dtype=torch.float32, device=qkv.device)
    lse = torch.empty((n, heads, L), dtype=torch.float32, device=qkv.device)
    stream = torch.cuda.current_stream(qkv.device)
    rc = _lib.on_device(qkv.device, _lib.lib.ps_vit_attention_forward, n, L, heads, inner // heads,
                        ctypes.c_void_p(qkv.data_ptr()), ctypes.c_float(scale), ctypes.c_void_p(out.data_ptr()),
                        ctypes.c_void_p(lse.data_ptr()), ctypes.c_void_p(stream.cuda_stream))
    _lib.check(rc, "ps_vit_attention_forward")
    return out, lse


def backward(qkv: Tensor, out: Tensor, d_out: Tensor, lse: Tensor, heads: int, scale: float) -> Tensor:
    """d_qkv [n, L, 3 * heads * 64] from the forward's (out, lse) and d_out = dL/dout."""
    n, L, three_inner = qkv.shape
    dim_head = three_inner // (3 * heads)
    ws = torch.empty(workspace_bytes(n, L, heads, dim_head), dtype=torch.uint8, device=qkv.device)
    d_qkv = torch.empty_like(qkv)
    stream = torch.cuda.current_stream(qkv.device)
    rc = _lib.on_device(qkv.device, _lib.lib.ps_vit_attention_backward, n, L, heads, dim_head,
                        ctypes.c_void_p(qkv.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                        ctypes.c_void_p(d_out.data_ptr()), ctypes.c_void_p(lse.data_ptr()), ctypes.c_float(scale),
                        ctypes.c_void_p(d_qkv.data_ptr()), ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                        ctypes.c_void_p(stream.cuda_stream))
    _lib.check(rc, "ps_vit_attention_backward")
    return d_qkv


class _VitAttention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv: Tensor, heads: int, scale: float):
        qkv = qkv.contiguous()
        out, lse = forward(qkv, heads, scale)
        ctx.save_for_backward(qkv, out, lse)
        ctx.heads, ctx.scale = heads, scale
        return out

    @staticmethod
    def backward(ctx, d_out: Tensor):
        qkv, out, lse = ctx.saved_tensors
        return backward(qkv, out, d_out.contiguous().float(), lse, ctx.heads, ctx.scale), None, None


def vit_attention(qkv: Tensor, heads: int, scale: float) -> Tensor:
    """qkv [n, L, 3 * heads * 64] (DINO's `qkv(x)`) -> softmax(q k^T * scale) v as [n, L, heads * 64]."""
    return _VitAttention.apply(qkv, heads, scale)
