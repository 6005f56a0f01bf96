"""The float64 restatement of the dense attention kernels (tests/attention_f64.py) and its bars, without a GPU.

- On operands that are already TF32 values the restatement is float64 autograd of softmax(q k^T scale) v.
- A numpy emulation of each kernel's arithmetic (its TF32 and float32 rounding points, float32 results of
  float64 products) stays within half of every bar over every input family.
- Five defects planted in the emulation each exceed their bar at least twice over on some family: D formed from
  the float32 dO, the row sum over unrounded P, a key past L left unmasked (a zero-filled key with logit 0), the
  row statistics shifted by one row at a 64-row boundary, and dK / dV of two heads swapped.
"""
import numpy as np
import pytest
import torch

from tests import attention_f64 as af

f32 = np.float32
LOG2E32 = f32(1.4426950408889634)
LN2_32 = f32(0.6931471805599453)
VIT_LS = (1, 7, 64, 65, 129)
DEFECTS = ("fp32_D", "unrounded_sum", "unmasked_key", "stats_shift", "head_swap")


def _tf32(a):
    return af._tf32(torch.from_numpy(np.ascontiguousarray(a, f32))).numpy()


def _mm(a, b):
    """float32 result of a float64 product (the emulation's stand-in for a float32 accumulation)."""
    return (a.astype(np.float64) @ b.astype(np.float64)).astype(f32)


def _exp2(x):
    return np.exp2(x.astype(np.float64)).astype(f32)


def _fma(a, b, c):
    return (a.astype(np.float64) * b + c).astype(f32)


def _split(x, heads):
    return af.split_heads(torch.from_numpy(x), heads).numpy()


def _merge(x, n):
    return af.merge_heads(torch.from_numpy(np.ascontiguousarray(x)), n).numpy()


def emulate(kind, qkv, d_out, heads, scale, defect=None):
    """The kernel's outputs (out, lse or stats, d_qkv) in the layout of its ABI, float32, with one planted defect."""
    qkv, d_out = qkv.numpy(), d_out.numpy()
    n, L, _ = qkv.shape
    q, k, v = (_tf32(_split(np.ascontiguousarray(t), heads)) for t in np.split(qkv, 3, -1))
    do_raw = _split(d_out, heads)
    do = _tf32(do_raw)
    B, _, d = q.shape
    sc = f32(scale)
    sl = f32(sc * LOG2E32)
    if kind == "sa":
        s = _mm(q, k.transpose(0, 2, 1))
        mb = (s.max(-1, keepdims=True) * sl).astype(f32)
        p_raw = _exp2(_fma(s, sl, -mb))
        p = _tf32(p_raw)
        tot = (p_raw if defect == "unrounded_sum" else p).astype(np.float64).sum(-1, keepdims=True).astype(f32)
        inv = (f32(1) / tot).astype(f32)
        out = (_mm(p, v) * inv).astype(f32)
        side = np.concatenate([mb, inv], -1)
        if defect == "stats_shift":
            side[:, 64:128] = side[:, 63:127].copy()
        mb_b, inv_b = side[..., :1], side[..., 1:]
        pn = (_tf32(_exp2(_fma(s, sl, -mb_b))) * inv_b).astype(f32)
        p_dv = _tf32(pn)
    else:
        m = np.full((B, L, 1), -np.inf, f32)
        l = np.zeros((B, L, 1), f32)
        o = np.zeros((B, L, d), f32)
        for k0 in range(0, L, af.VIT_TILE):
            kt, vt = k[:, k0:k0 + af.VIT_TILE], v[:, k0:k0 + af.VIT_TILE]
            st = (_mm(q, kt.transpose(0, 2, 1)) * sl).astype(f32)
            if defect == "unmasked_key" and kt.shape[1] < af.VIT_TILE:   # one zero-filled key past L, logit 0
                st = np.concatenate([st, np.zeros((B, L, 1), f32)], -1)
                vt = np.concatenate([vt, np.zeros((B, 1, d), f32)], 1)
            mx = np.maximum(m, st.max(-1, keepdims=True))
            a = _exp2((m - mx).astype(f32))
            p_raw = _exp2((st - mx).astype(f32))
            p = _tf32(p_raw)
            l = (l * a + (p_raw if defect == "unrounded_sum" else p).astype(np.float64).sum(-1, keepdims=True)).astype(f32)
            o = ((o * a).astype(f32) + _mm(p, vt)).astype(f32)
            m = mx
        out = (o * (f32(1) / l).astype(f32)).astype(f32)
        side = ((m + np.log2(l.astype(np.float64)).astype(f32)).astype(f32) * LN2_32).astype(f32)
        if defect == "stats_shift":
            side[:, 64:128] = side[:, 63:127].copy()
        s = (_mm(q, k.transpose(0, 2, 1)))
        lse2 = (side * LOG2E32).astype(f32)
        pn = _exp2(_fma(s, sl, -lse2))
        p_dv = _tf32(pn)
        side = side[..., 0]
    Dd = (do_raw if defect == "fp32_D" else do).astype(np.float64)
    D = (Dd * out).sum(-1, keepdims=True).astype(f32)
    dp = _mm(do, v.transpose(0, 2, 1))
    ds = _tf32((pn * (dp - D).astype(f32)).astype(f32) * sc)
    dq = _mm(ds, k)
    dk = _mm(ds.transpose(0, 2, 1), q)
    dv = _mm(p_dv.transpose(0, 2, 1), do)
    if defect == "head_swap":
        dk = dk.reshape(n, heads, L, d)[:, [1, 0] + list(range(2, heads))].reshape(B, L, d)
        dv = dv.reshape(n, heads, L, d)[:, [1, 0] + list(range(2, heads))].reshape(B, L, d)
    side = side.reshape((n, heads, L, 2) if kind == "sa" else (n, heads, L))
    d_qkv = np.concatenate([_merge(t, n) for t in (dq, dk, dv)], -1)
    return torch.from_numpy(_merge(out, n)), torch.from_numpy(np.ascontiguousarray(side)), torch.from_numpy(d_qkv)


def _case(kind, L, family, seed, heads=2, n=1):
    d = 64 if kind == "vit" else 128
    return af.make_inputs(family, n, L, heads, d, seed)


def _worst(kind, L, family, defect=None, heads=2):
    qkv, d_out, scale = _case(kind, L, family, 1000 + L, heads)
    res = af.restate(kind, qkv, d_out, heads, scale)
    return af.worst_ratios(kind, res, *emulate(kind, qkv, d_out, heads, scale, defect))


@pytest.mark.parametrize("kind,L", [("vit", 5), ("vit", 70), ("sa", 256)])
@pytest.mark.parametrize("scale", [0.125, 1.0])
def test_restatement_is_float64_autograd(kind, L, scale):
    heads, n = 2, 2
    d = 64 if kind == "vit" else 128
    g = torch.Generator().manual_seed(L)
    qkv = af._tf32(torch.randn(n, L, 3 * heads * d, generator=g))
    d_out = af._tf32(torch.randn(n, L, heads * d, generator=g))
    res = af.restate(kind, qkv, d_out, heads, scale)
    x = qkv.double().requires_grad_(True)
    q, k, v = (af.split_heads(t, heads) for t in x.chunk(3, -1))
    logits = q @ k.transpose(1, 2) * scale
    out = af.merge_heads(torch.softmax(logits, -1) @ v, n)
    out.backward(d_out.double())
    assert float((res.out - out.detach()).abs().max()) < 1e-12
    assert float((res.d_qkv - x.grad).abs().max()) < 1e-12
    lse = torch.logsumexp(logits.detach(), -1).reshape(n, heads, L)
    if kind == "vit":
        assert float((res.lse - lse).abs().max()) < 1e-12
    else:
        mx = logits.detach().amax(-1).reshape(n, heads, L)
        assert float((res.stats[..., 0] - mx * af.LOG2E).abs().max()) < 1e-12
        assert float((res.stats[..., 1] - torch.exp(mx - lse)).abs().max() / res.stats[..., 1].max()) < 1e-12


@pytest.mark.parametrize("family", list(af.FAMILIES))
@pytest.mark.parametrize("kind,L", [("vit", L) for L in VIT_LS] + [("sa", 256)])
def test_emulated_kernel_within_half_of_every_bar(kind, L, family):
    worst = _worst(kind, L, family)
    assert max(worst.values()) <= 0.5, worst


# defect -> kernels it applies to (the self-attention has no key mask: it always sees 256 valid keys)
PLANTED = [(kind, defect) for defect in DEFECTS for kind in ("vit", "sa") if not (kind == "sa" and defect == "unmasked_key")]


@pytest.mark.parametrize("kind,defect", PLANTED)
def test_planted_defect_exceeds_its_bar(kind, defect):
    """Each planted defect exceeds twice its bar on at least one family (at L = 129 / 256, so that a 64-row
    boundary and a partial key tile exist)."""
    L = 129 if kind == "vit" else 256
    best = {}
    for family in af.FAMILIES:
        best[family] = max(_worst(kind, L, family, defect).values())
        if best[family] >= 2.0:
            return
    pytest.fail(f"{kind} {defect}: worst error / bar per family {best}")
