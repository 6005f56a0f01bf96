"""The ViT flash attention (csrc/vit_attention.cu) and the 256-token self-attention (csrc/self_attention_tc.cu) at
their C ABIs, against the float64 restatement tests/attention_f64.py with its per-entry bars, across the descriptor
space the ABIs accept.

  1. ViT: L in {1, 2, 63, 64, 65, 127, 128, 129, 192, 257, 1025, 4097, 16384}, heads in {1, 6, 12, 16} and
     n in {1, 3, 14}, every (L, heads) pair with n cycling so that every (L, n) and (heads, n) pair occurs too; plus
     one call at n = 65535 (the grid.z limit), L = 1, one head.
  2. Self-attention: heads in {1, 2, 4, 7, 16} x n in {1, 3, 37}, plus every input family at 2 heads x 3 images.
  3. Input families (attention_f64.FAMILIES), cycled over the shapes: randn; V with a common offset; Q or K with
     a common offset; near-uniform and peaked rows, the one-hot construction; dO with an offset; scale 0.125,
     128^-0.5, 1 and 1e-3.
  4. Every entry of out, lse / stats and d_qkv within its bar; the failure names the image, head, token, channel,
     CTA and warpgroup of the worst entry.
  5. Canaries: outputs, row statistics and gradients in NaN-filled buffers followed by guard words (every entry
     written, no guard touched); inputs are views in front of tails of NaN in one run and of 3e38 in the other,
     and both runs give the same bits (so nothing past the tensors is read, and repeated calls are bitwise equal).

Measured on an NVIDIA H100 80GB HBM3 (700 W power limit): see DESIGN.md section 6 for the worst ratio per kernel,
tensor and family.
"""
import ctypes

import pytest
import torch

from pixelsplat_b200 import _lib
from tests import attention_f64 as af

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FAMILIES = list(af.FAMILIES)
GUARD = 64                                   # guard words after every output
GUARD_VALUE = -1.2345e-20

VIT_L = (1, 2, 63, 64, 65, 127, 128, 129, 192, 257, 1025, 4097, 16384)
VIT_H = (1, 6, 12, 16)
VIT_N = (1, 3, 14)
VIT_CASES = [(L, h, VIT_N[(i - j) % 3], FAMILIES[(4 * i + j) % len(FAMILIES)])
             for i, L in enumerate(VIT_L) for j, h in enumerate(VIT_H)] + [(1, 1, 65535, "randn")]
SA_CASES = [(h, n, FAMILIES[(3 * i + j) % len(FAMILIES)]) for i, h in enumerate((1, 2, 4, 7, 16))
            for j, n in enumerate((1, 3, 37))] + [(2, 3, f) for f in FAMILIES]


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _guarded(shape):
    """A NaN-filled tensor of `shape` at the front of a buffer whose GUARD trailing words hold GUARD_VALUE."""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + GUARD,), float("nan"), device=DEV)
    buf[n:] = GUARD_VALUE
    return buf[:n].view(shape), buf


def _tailed(x, fill):
    """x copied to the front of a buffer followed by 4096 words of `fill`, as a view of x's shape."""
    buf = torch.full((x.numel() + 4096,), fill, device=DEV)
    buf[:x.numel()] = x.reshape(-1)
    return buf[:x.numel()].view_as(x)


def _run(kind, qkv, d_out, heads, scale):
    """One forward and one backward at the ABI into guarded NaN-filled outputs: (out, side, d_qkv), guard buffers."""
    n, L, _ = qkv.shape
    d = 64 if kind == "vit" else 128
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    out, b_out = _guarded((n, L, heads * d))
    side, b_side = _guarded((n, heads, L) if kind == "vit" else (n, heads, L, 2))
    d_qkv, b_dqkv = _guarded(tuple(qkv.shape))
    if kind == "vit":
        _lib.check(_lib.lib.ps_vit_attention_forward(n, L, heads, d, _p(qkv), ctypes.c_float(scale), _p(out),
                                                     _p(side), st), "forward")
        ws_bytes = ctypes.c_size_t()
        _lib.check(_lib.lib.ps_vit_attention_backward_workspace_bytes(n, L, heads, d, ctypes.byref(ws_bytes)), "ws")
        ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=DEV)
        _lib.check(_lib.lib.ps_vit_attention_backward(n, L, heads, d, _p(qkv), _p(out), _p(d_out), _p(side),
                                                      ctypes.c_float(scale), _p(d_qkv), _p(ws), ws.numel(), st),
                   "backward")
    else:
        _lib.check(_lib.lib.ps_self_attention_forward_stats(n, L, heads, d, _p(qkv), ctypes.c_float(scale), _p(out),
                                                            _p(side), st), "forward")
        _lib.check(_lib.lib.ps_self_attention_backward(n, L, heads, d, _p(qkv), _p(out), _p(d_out), _p(side),
                                                       ctypes.c_float(scale), _p(d_qkv), st), "backward")
    torch.cuda.synchronize()
    return (out, side, d_qkv), (b_out, b_side, b_dqkv)


def _sweep(kind, n, L, heads, family, seed):
    d = 64 if kind == "vit" else 128
    qkv, d_out, scale = af.make_inputs(family, n, L, heads, d, seed)
    qkv, d_out = qkv.to(DEV), d_out.to(DEV)
    runs = []
    for fill in (float("nan"), 3e38):
        results, guards = _run(kind, _tailed(qkv, fill), _tailed(d_out, fill), heads, scale)
        for name, t, g in zip(("out", "row statistics", "d_qkv"), results, guards):
            assert not t.isnan().any(), f"{name}: {int(t.isnan().sum())} entries never written"
            assert bool((g[t.numel():] == GUARD_VALUE).all()), f"{name}: a guard word past the tensor was written"
        runs.append(results)
    for name, a, b in zip(("out", "row statistics", "d_qkv"), *runs):
        assert torch.equal(a, b), f"{name}: the NaN-tail and 3e38-tail runs differ"
    res = af.restate(kind, qkv, d_out, heads, scale)
    worst = af.check_all(kind, res, *runs[0])
    print(f"{kind} n={n} L={L} heads={heads} {family}: " + " ".join(f"{k} {v:.3f}" for k, v in worst.items()))


@pytest.mark.parametrize("L,heads,n,family", VIT_CASES, ids=[f"L{L}-h{h}-n{n}-{f}" for L, h, n, f in VIT_CASES])
def test_vit_attention_within_bars(L, heads, n, family):
    _sweep("vit", n, L, heads, family, seed=L * 1000 + heads * 100 + n)


@pytest.mark.parametrize("heads,n,family", SA_CASES, ids=[f"h{h}-n{n}-{f}" for h, n, f in SA_CASES])
def test_self_attention_within_bars(heads, n, family):
    _sweep("sa", n, 256, heads, family, seed=heads * 100 + n)
