"""GPU tests of the flash-style ViT attention kernel (csrc/vit_attention.cu) against DINO's formula
softmax(q k^T * scale) v evaluated in float64 by torch, at DINO's token counts (the CLS token makes them odd).

Stated tolerance: q, k, v, the probabilities, dO and dS are rounded to the nearest TF32 (10 explicit mantissa bits)
before the tensor cores see them; accumulation is fp32.  The bar against float64 is 2e-3 relative (max-norm over
the tensor) on the output and on each of dQ, dK, dV, the same as the 256-token self-attention kernel's; lse
carries the logits' TF32 error and is within 2e-3 absolute.  At L = 1 the exact dQ and dK are 0 (a one-key soft-max
is constant); there they are held to 2e-3 of dV's largest entry.  Measured on an H100 over CASES: output <= 1.1e-3,
dQ / dK / dV <= 1.2e-3 (both at L = 4097; <= 1.0e-3 up to L = 1025), lse <= 9.3e-4.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
D = 64

CASES = [(L, n, h) for L in (1, 7, 64, 65, 257, 1025) for (n, h) in ((1, 6), (14, 12))] + \
    [(4097, 1, 6), (4097, 1, 12)]


def _split(qkv, heads):
    n, L, _ = qkv.shape
    return [t.reshape(n, L, heads, D).transpose(1, 2) for t in qkv.chunk(3, dim=-1)]   # [n, H, L, 64]


def _reference(qkv, d_out, heads, scale):
    """float64 output, lse and d_qkv of DINO's explicit attention."""
    n, L, _ = qkv.shape
    x = qkv.double().requires_grad_(True)
    q, k, v = _split(x, heads)
    s = (q @ k.transpose(-1, -2)) * scale
    lse = torch.logsumexp(s, -1)
    out = (s.softmax(-1) @ v).transpose(1, 2).reshape(n, L, heads * D)
    out.backward(d_out.double())
    return out.detach(), lse.detach(), x.grad


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


def _inputs(L, n, heads, seed):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(n, L, 3 * heads * D, generator=g).to(DEV)
    d_out = torch.randn(n, L, heads * D, generator=g).to(DEV)
    return qkv, d_out


@pytest.mark.parametrize("L,n,heads", CASES)
def test_matches_float64(L, n, heads):
    from pixelsplat_b200.encoder import vit_attention as va
    qkv, d_out = _inputs(L, n, heads, L * 100 + n * 10 + heads)
    scale = D ** -0.5
    out, lse = va.forward(qkv, heads, scale)
    d_qkv = va.backward(qkv, out, d_out, lse, heads, scale)
    torch.cuda.synchronize()
    ref_out, ref_lse, ref_d = _reference(qkv, d_out, heads, scale)
    assert _rel(out, ref_out) < 2e-3
    assert float((lse.double() - ref_lse).abs().max()) < 2e-3
    dv_scale = float(ref_d.chunk(3, -1)[2].abs().max())
    for got, ref in zip(d_qkv.chunk(3, -1), ref_d.chunk(3, -1)):
        scale_ref = float(ref.abs().max()) if L > 1 else dv_scale
        assert float((got.double() - ref).abs().max()) < 2e-3 * scale_ref


def test_memory_past_the_tensors_has_no_influence():
    """qkv and d_out are views at the front of larger buffers; the tail holds NaN in one run and huge values in
    the other.  Both runs must give the same bits, so no key, query or gradient row past L is ever read."""
    from pixelsplat_b200.encoder import vit_attention as va
    L, n, heads = 65, 2, 6
    qkv, d_out = _inputs(L, n, heads, 5)
    results = []
    for fill in (float("nan"), 3e38):
        big = torch.full((qkv.numel() + 4096,), fill, device=DEV)
        big[:qkv.numel()] = qkv.reshape(-1)
        bdo = torch.full((d_out.numel() + 4096,), fill, device=DEV)
        bdo[:d_out.numel()] = d_out.reshape(-1)
        x, dy = big[:qkv.numel()].view_as(qkv), bdo[:d_out.numel()].view_as(d_out)
        out, lse = va.forward(x, heads, 0.125)
        results.append((out, lse, va.backward(x, out, dy, lse, heads, 0.125)))
    for a, b in zip(*results):
        assert torch.isfinite(a).all() and torch.equal(a, b)


def test_structured_input_catches_layout_errors():
    """One-hot attention per head: query i of head h matches key perm_h[i] overwhelmingly, so out[i, h] equals
    v[perm_h[i], h]; a swapped head, token tile or channel group shows up as a wrong row."""
    from pixelsplat_b200.encoder import vit_attention as va
    L, n, heads = 257, 2, 6
    g = torch.Generator().manual_seed(7)
    q = torch.zeros(n, L, heads, D)
    k = torch.zeros(n, L, heads, D)
    perms = [[torch.randperm(L, generator=g) for _ in range(heads)] for _ in range(n)]
    basis = torch.randn(L, D, generator=g)
    basis = basis / basis.norm(dim=-1, keepdim=True)
    for b in range(n):
        for h in range(heads):
            q[b, :, h] = 60.0 * basis[perms[b][h]]
            k[b, :, h] = basis
    v = torch.randn(n, L, heads, D, generator=g)
    qkv = torch.cat([q.reshape(n, L, -1), k.reshape(n, L, -1), v.reshape(n, L, -1)], -1).to(DEV)
    out, _ = va.forward(qkv, heads, 1.0)
    expect = torch.stack([torch.stack([v[b, perms[b][h], h] for h in range(heads)], 1) for b in range(n)])
    assert float((out.cpu().reshape(n, L, heads, D) - expect).abs().max()) < 2e-2


def test_backward_is_bitwise_repeatable():
    from pixelsplat_b200.encoder import vit_attention as va
    qkv, d_out = _inputs(1025, 3, 12, 11)
    out, lse = va.forward(qkv, 12, 0.125)
    a = va.backward(qkv, out, d_out, lse, 12, 0.125)
    b = va.backward(qkv, out, d_out, lse, 12, 0.125)
    assert torch.equal(a, b)


def test_cuda_graph_capture_and_replay():
    from pixelsplat_b200.encoder import vit_attention as va
    heads, scale = 6, 0.125
    qkv, d_out = _inputs(257, 2, heads, 13)
    x = qkv.clone().requires_grad_(True)
    va.vit_attention(x, heads, scale).backward(d_out)                    # warm-up: attributes, allocator
    x.grad = None
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph):
            y = va.vit_attention(x, heads, scale)
            y.backward(d_out)
    torch.cuda.current_stream().wait_stream(s)
    new_qkv, _ = _inputs(257, 2, heads, 14)
    with torch.no_grad():
        x.copy_(new_qkv)
    graph.replay()
    torch.cuda.synchronize()
    ref = new_qkv.clone().requires_grad_(True)
    ref_y = va.vit_attention(ref, heads, scale)
    ref_y.backward(d_out)
    assert torch.equal(y, ref_y) and torch.equal(x.grad, ref.grad)


def test_autograd_function_matches_the_explicit_formula():
    """The autograd route (what DINO's Attention calls) against the fp32 torch formula it replaces."""
    from pixelsplat_b200.encoder import vit_attention as va
    heads, scale = 12, D ** -0.5
    qkv, d_out = _inputs(1025, 2, heads, 17)
    x = qkv.clone().requires_grad_(True)
    va.vit_attention(x, heads, scale).backward(d_out)
    ref_out, _, ref_d = _reference(qkv, d_out, heads, scale)
    assert _rel(x.grad, ref_d) < 2e-3
