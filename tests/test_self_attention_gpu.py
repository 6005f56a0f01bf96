"""GPU tests of the wgmma self-attention kernels (csrc/self_attention_tc.cu, SURVEY.md 8 row a14)
against the reference's formula softmax(q k^T * scale) v
(/root/reference/src/model/transformer/attention.py:54-70, z = None) evaluated in float64 by torch.

Stated tolerance: the operands (q, k, v and the un-normalised probabilities) are rounded to the
nearest TF32 (10 explicit mantissa bits) before the tensor cores see them; accumulation is fp32.
Against float64 the bar is 2e-3 (relative, max-norm) on the logits and on the output; against a
float64 evaluation of the SAME rounded operands -- which isolates layout / indexing mistakes from
rounding -- it is 2e-5 on the logits.
"""
import ctypes

import pytest
import torch

from tests.attention_f64 import _tf32

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _split(qkv, heads):
    n, L, _ = qkv.shape
    return [t.reshape(n, L, heads, -1).transpose(1, 2) for t in qkv.chunk(3, dim=-1)]


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.mark.parametrize("n,heads", [(1, 4), (3, 4), (2, 1), (5, 8)])
def test_logits_and_output_match_float64(n, heads):
    from pixelsplat_b200.encoder import self_attention_tc as sa
    g = torch.Generator().manual_seed(n * 10 + heads)
    qkv = torch.randn(n, 256, 3 * heads * 128, generator=g).to(DEV)
    scale = 128 ** -0.5
    q, k, v = _split(qkv, heads)
    s64 = q.double() @ k.double().transpose(-1, -2)
    s_tc = sa.qk_logits_tc(qkv, heads)
    assert _rel(s_tc, s64) < 2e-3
    s_trunc = _tf32(q).double() @ _tf32(k).double().transpose(-1, -2)
    assert _rel(s_tc, s_trunc) < 2e-5
    out = sa.self_attention_tc(qkv, heads, scale)
    ref = (torch.softmax(s64 * scale, -1) @ v.double()).transpose(1, 2).reshape(n, 256, -1)
    assert out.shape == ref.shape
    assert _rel(out, ref) < 2e-3
    # every (image, head, row) is a convex combination of that head's values: catches a swapped half / head
    lo = v.amin(dim=2).transpose(0, 1).reshape(heads, n, 1, 128)
    o4 = out.reshape(n, 256, heads, 128).permute(2, 0, 1, 3)
    assert (o4 >= lo - 1e-3).all() and (o4 <= v.amax(dim=2).transpose(0, 1).reshape(heads, n, 1, 128) + 1e-3).all()


def test_structured_input_catches_layout_errors():
    """One-hot attention: query i matches key perm[i] overwhelmingly, so out[i] == v[perm[i]]."""
    from pixelsplat_b200.encoder import self_attention_tc as sa
    heads, n = 4, 2
    g = torch.Generator().manual_seed(3)
    basis = torch.linalg.qr(torch.randn(256, 256, generator=g))[0][:, :128] * 40.0      # 256 distinct directions
    qkv = torch.zeros(n, 256, 3, heads, 128)
    perms = torch.stack([torch.stack([torch.randperm(256, generator=g) for _ in range(heads)]) for _ in range(n)])
    for i in range(n):
        for h in range(heads):
            qkv[i, :, 1, h] = basis
            qkv[i, :, 0, h] = basis[perms[i, h]]
    qkv[:, :, 2] = torch.randn(n, 256, heads, 128, generator=g)
    x = qkv.reshape(n, 256, -1).to(DEV)
    out = sa.self_attention_tc(x, heads, 1.0).reshape(n, 256, heads, 128).cpu()
    q, k, v = _split(x, heads)
    ref = (torch.softmax(q.double() @ k.double().transpose(-1, -2), -1) @ v.double()).transpose(1, 2).cpu()
    assert _rel(out, ref) < 2e-3
    # and the structure really is a permutation for most rows
    hit = 0
    for i in range(n):
        for h in range(heads):
            hit += int(((out[i, :, h] - qkv[i, perms[i, h], 2, h]).abs().amax(-1) < 5e-2).sum())
    assert hit > 0.9 * n * heads * 256


@pytest.mark.parametrize("n,heads", [(2, 4), (1, 1), (3, 8)])
def test_gradients_match_float64(n, heads):
    """The wgmma backward: dq, dk, dv separately against float64 autograd of the reference formula.  Stated
    tolerance: TF32 operands (q, k, v, dO, probabilities and d score rounded to 10 mantissa bits) -> 3e-3
    relative (max-norm) per tensor."""
    from pixelsplat_b200 import _lib
    from pixelsplat_b200.encoder import self_attention_tc as sa
    scale = 128 ** -0.5
    g = torch.Generator().manual_seed(11 + n)
    qkv = torch.randn(n, 256, 3 * heads * 128, generator=g).to(DEV).requires_grad_(True)
    w = torch.randn(n, 256, heads * 128, generator=g).to(DEV)
    q, k, v = _split(qkv.double(), heads)
    ref = (torch.softmax(q @ k.transpose(-1, -2) * scale, -1) @ v).transpose(1, 2).reshape(n, 256, -1)
    (ref * w.double()).sum().backward()
    g_ref = qkv.grad.clone(); qkv.grad = None
    before = _lib.lib.ps_launch_count()
    (sa.self_attention_tc(qkv, heads, scale) * w).sum().backward()
    assert _lib.lib.ps_launch_count() == before + 2                      # one forward, one backward kernel
    g_tc = qkv.grad.clone(); qkv.grad = None
    for name, a, b in zip("qkv", g_tc.chunk(3, dim=-1), g_ref.chunk(3, dim=-1)):
        assert _rel(a, b) < 3e-3, (name, _rel(a, b))
        for h in range(heads):                                               # per head: catches a swapped head / half
            sl = slice(h * 128, (h + 1) * 128)
            assert _rel(a[..., sl], b[..., sl]) < 5e-3, (name, h)
            assert _rel(a[:, :128, sl], b[:, :128, sl]) < 5e-3 and _rel(a[:, 128:, sl], b[:, 128:, sl]) < 5e-3


def test_backward_differentiates_the_forward_that_ran():
    """Finite differences of the KERNEL's own forward along a random direction agree with its backward (the
    probabilities are rebuilt from the saved row statistics, not recomputed in another precision)."""
    from pixelsplat_b200.encoder import self_attention_tc as sa
    heads, n, scale = 4, 1, 128 ** -0.5
    g = torch.Generator().manual_seed(5)
    qkv = (torch.randn(n, 256, 3 * heads * 128, generator=g) * 0.5).to(DEV).requires_grad_(True)
    w = torch.randn(n, 256, heads * 128, generator=g).to(DEV)
    d = torch.randn(n, 256, 3 * heads * 128, generator=g).to(DEV)
    (sa.self_attention_tc(qkv, heads, scale) * w).sum().backward()
    analytic = float((qkv.grad * d).sum())
    # float64 central difference of the float64 formula as the yardstick for the directional derivative
    with torch.no_grad():
        f = lambda x: float(((torch.softmax(_split(x, heads)[0] @ _split(x, heads)[1].transpose(-1, -2) * scale, -1)
                              @ _split(x, heads)[2]).transpose(1, 2).reshape(n, 256, -1) * w.double()).sum())
        eps = 1e-4
        fd = (f(qkv.double() + eps * d.double()) - f(qkv.double() - eps * d.double())) / (2 * eps)
    assert abs(analytic - fd) <= 3e-3 * max(abs(fd), 1.0), (analytic, fd)


def test_module_uses_the_kernel_and_matches_fp32(monkeypatch):
    from pixelsplat_b200 import _lib
    from pixelsplat_b200.encoder.transformer import Attention
    torch.manual_seed(0)
    att = Attention(128, heads=4, dim_head=128, selfatt=True).to(DEV)
    x = torch.randn(6, 256, 128, device=DEV)
    before = _lib.lib.ps_launch_count()
    y_tc = att(x)
    assert _lib.lib.ps_launch_count() == before + 1
    monkeypatch.setenv("PIXELSPLAT_B200_SELF_ATTENTION", "fp32")
    y_32 = att(x)
    assert _lib.lib.ps_launch_count() == before + 1
    assert _rel(y_tc, y_32) < 2e-3
    # a shape the kernel is not written for goes through torch
    assert att(torch.randn(2, 64, 128, device=DEV)).shape == (2, 64, 128)


def test_unsupported_shape_is_an_error_at_the_abi():
    from pixelsplat_b200 import _lib
    buf = torch.zeros(1 << 20, device=DEV)
    rc = _lib.lib.ps_self_attention_forward(1, 128, 4, 128, ctypes.c_void_p(buf.data_ptr()), ctypes.c_float(1.0),
                                            ctypes.c_void_p(buf.data_ptr()), 0, None)
    assert rc == 3 and b"256 tokens" in _lib.lib.ps_last_error()
