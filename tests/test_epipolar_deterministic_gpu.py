"""The epipolar attention backward under torch.use_deterministic_algorithms(True)
(include/pixelsplat_b200.h ps_epipolar_attention_backward_deterministic: a fixed-order d(feature map)).

  1. Bit-identical repeats of _EpipolarAttentionFn's backward: heads 1-4, S in {1, 7, 32}, pe_dim 0 / 20, v = 2 / 3
     with the view-embedding bias, b = 2, grids 8x8 and 6x10, the generic / parallel / diverging rigs, a rig whose
     epipole lies inside the other image (long cell lists) and configs[2] at batch 1.
  2. The same answer as with the flag off: dqt, dpq, dbias bit-identical; dfeat within 1e-6 norm-wise, and no
     further from a float64 restatement than 1.5x the float-atomic path.
  3. The module bars of tests/test_epipolar_gpu.py hold with the flag on.
  4. A CUDA graph of an EpipolarTransformer forward + backward captured with the flag on replays the eager step.
  5. A small configs[2]-style training step (encoder, tail, fused MSE + LossDepth + SSIM) repeats bit for bit.
  6. With the flag off the backward calls the float-atomic entry point only.
"""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import golden_util as gu
from tests import test_epipolar_gpu as epi_gpu

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture
def det():
    """torch's deterministic flag on for the test; the flag and the cuBLAS workspace setting torch asks for under the
    flag are restored afterwards, also when the test fails."""
    flag, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    cublas = os.environ.get("CUBLAS_WORKSPACE_CONFIG")
    os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(flag, warn_only=warn_only)
        if cublas is None:
            os.environ.pop("CUBLAS_WORKSPACE_CONFIG", None)
        else:
            os.environ["CUBLAS_WORKSPACE_CONFIG"] = cublas


def _case(b, v, grid, S, heads, npe, rig, bias=True, seed=0):
    """Inputs of _EpipolarAttentionFn and the output cotangents (seeded)."""
    from pixelsplat_b200.encoder.attention_fused import epipolar_geometry
    ext, K, near, far = [t.to(DEV, torch.float32) for t in gu.camera_rig(b, v, rig)]
    geom = epipolar_geometry(ext, K, near, far, grid, S)
    h, w = grid
    n, ov = b * v * h * w, v - 1
    g = torch.Generator().manual_seed(1000 + seed)
    r = lambda *s, scale=1.0: (torch.randn(s, generator=g) * scale).to(DEV)
    x = dict(qt=r(n, heads, 128, scale=0.3), pq=r(n, heads, npe, scale=0.3), bias=r(n, heads, ov) if bias else None,
             feat=r(b, v, h, w, 128), dz=r(n, heads, 128), de=r(n, heads, npe),
             dmass=r(n, heads, ov) if bias else None)
    return geom, heads, x


def _backward(geom, heads, x):
    """(dqt, dpq, dbias, dfeat) of one _EpipolarAttentionFn forward + backward, in the flag's current mode."""
    from pixelsplat_b200.encoder.attention_fused import _EpipolarAttentionFn
    leaves = {k: x[k].clone().requires_grad_(True) for k in ("qt", "pq", "bias", "feat") if x[k] is not None}
    z, e, mass = _EpipolarAttentionFn.apply(leaves["qt"], leaves["pq"], leaves.get("bias"), leaves["feat"], geom, heads)
    outs, cots = [z, e], [x["dz"], x["de"]]
    if x["bias"] is not None:
        outs.append(mass)
        cots.append(x["dmass"])
    grads = torch.autograd.grad(outs, list(leaves.values()), cots)
    got = dict(zip(leaves, grads))
    return got["qt"], got["pq"], got.get("bias"), got["feat"]


def _longest_cell_list(geom, S, grid):
    """Slots per bilinear cell, restated in torch from the geometry (the kernel's cell key; diagnostics only)."""
    h, w = grid
    seg, valid = geom.segments, geom.valid.bool()
    b, v, ov, R, _ = seg.shape
    u = (torch.arange(S, device=seg.device, dtype=torch.float32) + 0.5) / S
    sx = seg[..., None, 0] + u * (seg[..., None, 2] - seg[..., None, 0])
    sy = seg[..., None, 1] + u * (seg[..., None, 3] - seg[..., None, 1])
    bx = torch.floor(sx * w - 0.5).clamp(-2, w + 1)
    by = torch.floor(sy * h - 0.5).clamp(-2, h + 1)
    vi = torch.arange(v, device=seg.device)[:, None]
    o = torch.arange(ov, device=seg.device)[None, :]
    other = torch.where(o < vi, o, o + 1)                                       # [v, ov]
    m = torch.arange(b, device=seg.device)[:, None, None] * v + other[None]    # [b, v, ov]
    key = (m[..., None, None] * (h + 1) + by + 1) * (w + 1) + bx + 1
    ok = valid[..., None] & (bx >= -1) & (bx < w) & (by >= -1) & (by < h)
    counts = torch.bincount(key[ok].long().flatten(), minlength=b * v * (h + 1) * (w + 1))
    return int(counts.max()), float(counts[counts > 0].float().mean())


def _reference_f64(geom, heads, x):
    """Float64 restatement of the fused attention (grid_sample sampling, PE, soft-max over all (ov, s)) and autograd:
    d(feature map).  The flag must be off (grid_sample's backward has no deterministic implementation)."""
    b, v, h, w, C = x["feat"].shape
    ov, S, R = v - 1, geom.samples, h * w
    npe = x["pq"].shape[-1]
    feat = x["feat"].double().requires_grad_(True)
    fmap = feat.permute(0, 1, 4, 2, 3)                                          # [b, v, C, h, w]
    u = (torch.arange(S, device=DEV, dtype=torch.float64) + 0.5) / S
    seg = geom.segments.double()
    xy = seg[..., None, :2] + u[:, None] * (seg[..., None, 2:] - seg[..., None, :2])   # [b, v, ov, R, S, 2]
    samples = []
    for vi in range(v):
        per = []
        for o in range(ov):
            other = o if o < vi else o + 1
            grid = (2 * xy[:, vi, o] - 1).reshape(b, R * S, 1, 2)
            smp = F.grid_sample(fmap[:, other], grid, mode="bilinear", padding_mode="zeros", align_corners=False)
            per.append(smp[..., 0].permute(0, 2, 1).reshape(b, R, S, C))
        samples.append(torch.stack(per, 1))
    f = torch.stack(samples, 1) * geom.valid[..., None, None].double()           # [b, v, ov, R, S, C]
    f = f.permute(0, 1, 3, 2, 4, 5).reshape(b * v * R, ov, S, C)
    rd = geom.rel_disparity.double().permute(0, 1, 3, 2, 4).reshape(b * v * R, ov, S)
    freq = float(np.float32(2 * math.pi)) * 2.0 ** torch.arange(npe // 2, device=DEV, dtype=torch.float64)
    ph = rd[..., None] * freq
    pe = torch.stack([torch.sin(ph), torch.sin(ph + math.pi / 2)], -1).reshape(*rd.shape, npe)
    qt, pq = x["qt"].double(), x["pq"].double()
    score = torch.einsum("nhc,nosc->nhos", qt, f) + torch.einsum("nhj,nosj->nhos", pq, pe)
    if x["bias"] is not None:
        score = score + x["bias"].double()[..., None]
    n = score.shape[0]
    a = torch.softmax(score.reshape(n, heads, ov * S), -1).reshape(n, heads, ov, S)
    z = torch.einsum("nhos,nosc->nhc", a, f)
    e = torch.einsum("nhos,nosj->nhj", a, pe)
    loss = (z * x["dz"].double()).sum() + (e * x["de"].double()).sum()
    if x["bias"] is not None:
        loss = loss + (a.sum(-1) * x["dmass"].double()).sum()
    (g,) = torch.autograd.grad(loss, feat)
    return g


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300))


# (b, v, grid, S, heads, pe_dim, rig, bias)
CASES = {
    "h1-s1-pe0": (2, 2, (8, 8), 1, 1, 0, "generic", False),
    "h2-s7-pe20": (2, 2, (8, 8), 7, 2, 20, "generic", False),
    "h3-s32-pe20-v3": (2, 3, (8, 8), 32, 3, 20, "generic", True),
    "h4-s32-pe20": (2, 2, (8, 8), 32, 4, 20, "generic", False),
    "h4-s7-pe0-v3-6x10": (2, 3, (6, 10), 7, 4, 0, "generic", True),
    "h1-s32-pe20-6x10": (2, 2, (6, 10), 32, 1, 20, "generic", False),
    "h2-s32-pe20-parallel-v3": (2, 3, (8, 8), 32, 2, 20, "parallel", True),
    "h4-s32-pe20-diverging": (2, 2, (8, 8), 32, 4, 20, "diverging", False),
    "h3-s1-pe20-diverging-v3": (2, 3, (6, 10), 1, 3, 20, "diverging", True),
    "h4-s32-pe20-epipole": (2, 2, (16, 16), 32, 4, 20, "epipole", False),
    "h4-s32-pe20-epipole-v3": (2, 3, (16, 16), 32, 4, 20, "epipole", True),
    "config2-b1": (1, 2, (64, 64), 32, 4, 20, "generic", False),
}


@pytest.mark.parametrize("name", list(CASES))
def test_repeats_are_bit_identical(det, name):
    b, v, grid, S, heads, npe, rig, bias = CASES[name]
    geom, heads, x = _case(b, v, grid, S, heads, npe, rig, bias)
    runs = [_backward(geom, heads, x) for _ in range(3)]
    for other in runs[1:]:
        for i, (p, q) in enumerate(zip(runs[0], other)):
            assert (p is None and q is None) or torch.equal(p, q), (name, ("dqt", "dpq", "dbias", "dfeat")[i])
    assert torch.isfinite(runs[0][3]).all()
    assert (runs[0][3].abs().sum() > 0) == bool(geom.valid.any())      # the diverging rig can leave no valid ray
    if rig == "epipole":
        longest, mean = _longest_cell_list(geom, S, grid)
        print(name, "longest cell list", longest, "mean", mean)
        assert longest >= 4 * mean and longest > 4 * S      # a few cells hold the near ends of many segments


@pytest.mark.parametrize("name", ["h4-s32-pe20", "h3-s32-pe20-v3", "h4-s7-pe0-v3-6x10", "h2-s32-pe20-parallel-v3",
                                  "h4-s32-pe20-diverging", "h4-s32-pe20-epipole", "config2-b1"])
def test_same_answer_as_flag_off(name):
    b, v, grid, S, heads, npe, rig, bias = CASES[name]
    geom, heads, x = _case(b, v, grid, S, heads, npe, rig, bias)
    flag = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        on = _backward(geom, heads, x)
        torch.use_deterministic_algorithms(False)
        off = _backward(geom, heads, x)
    finally:
        torch.use_deterministic_algorithms(flag)
    for i in range(3):
        assert (on[i] is None and off[i] is None) or torch.equal(on[i], off[i]), ("dqt", "dpq", "dbias")[i]
    assert _rel(on[3], off[3]) < 1e-6, _rel(on[3], off[3])
    if name != "config2-b1":          # the float64 restatement materialises the samples: small cases only
        ref = _reference_f64(geom, heads, x)
        d_on, d_off = _rel(on[3], ref), _rel(off[3], ref)
        print(name, "dfeat vs float64: deterministic", d_on, "float atomics", d_off)
        assert d_on <= 1.5 * d_off, (d_on, d_off)


# ------------------------------------------------------------------ 3. module bars with the flag on
@pytest.mark.parametrize("v", [2, 3])
def test_epipolar_transformer_matches_reference(det, v, monkeypatch):
    epi_gpu.test_epipolar_transformer_matches_reference(v, monkeypatch)


def test_config2_shape_matches_reference(det):
    epi_gpu.test_config2_shape_matches_reference()


# ------------------------------------------------------------------ 4. CUDA graph
def test_cuda_graph_replay_matches_eager(det):
    m = epi_gpu._modules(2)
    feats, ext, K, near, far, wgt = epi_gpu._inputs(2)
    params = [feats] + list(m.parameters())

    def step():
        for p in params:
            p.grad = None
        out, _ = m(feats, ext, K, near, far)
        (out * wgt).sum().backward()
        return out.detach(), [p.grad for p in params]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
        eager = step()
        eager = (eager[0].clone(), [None if g is None else g.clone() for g in eager[1]])
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out[0], eager[0])
        for a, b in zip(out[1], eager[1]):
            assert (a is None and b is None) or torch.equal(a, b)


# ------------------------------------------------------------------ 5. end to end
def test_training_step_is_bit_identical(det):
    """EpipolarTransformer -> EncoderEpipolarTail -> DecoderSplattingCUDA.forward_mse (fused depth) + LossDepth +
    (1 - SSIM) -> backward, twice: the loss, every parameter gradient and the input features' gradient."""
    from pixelsplat_b200 import loss as L
    from pixelsplat_b200 import synthetic
    from pixelsplat_b200.decoder import DecoderSplattingCUDA, DecoderSplattingCUDACfg
    from pixelsplat_b200.encoder import EpipolarTransformer, EpipolarTransformerCfg, ImageSelfAttentionCfg
    from pixelsplat_b200.encoder.encoder_tail import EncoderEpipolarTail, EncoderTailCfg
    B, T, HW = 1, 2, 64
    torch.manual_seed(0)
    cfg = EpipolarTransformerCfg(ImageSelfAttentionCfg(4, 10, 2, 4, 128, 128, 256), 10, 2, 4, 32, 128, 256, 4)
    enc = EpipolarTransformer(cfg, 128, num_context_views=2).to(DEV)
    head = EncoderEpipolarTail(EncoderTailCfg()).to(DEV)
    dec = DecoderSplattingCUDA(DecoderSplattingCUDACfg("splatting_cuda"),
                               type("D", (), {"background_color": [0.0, 0.0, 0.0]})()).to(DEV)
    g = torch.Generator().manual_seed(1234)
    feats = torch.randn(B, 2, 128, HW, HW, generator=g).to(DEV)
    images = torch.rand(B, 2, 3, HW, HW, generator=g).to(DEV)
    ctx_e = torch.eye(4).repeat(B, 2, 1, 1)
    ctx_e[:, 1, 0, 3] = 1.0
    ctx_k = synthetic.intrinsics_re10k(2)[None].repeat(B, 1, 1, 1)
    near_v, far_v = synthetic.bounds_from_baseline(1.0, HW, HW, 3.0 * HW, 0.5)
    tgt_e = torch.stack([synthetic.target_cameras(T, seed=s) for s in range(B)]).to(DEV)
    tgt_k = synthetic.intrinsics_re10k(T)[None].repeat(B, 1, 1, 1).to(DEV)
    target = torch.rand(B, T, 3, HW, HW, generator=g).to(DEV)
    ctx_e, ctx_k = ctx_e.to(DEV), ctx_k.to(DEV)
    near_c, far_c = torch.full((B, 2), near_v, device=DEV), torch.full((B, 2), far_v, device=DEV)
    near_t, far_t = torch.full((B, T), near_v, device=DEV), torch.full((B, T), far_v, device=DEV)
    context = dict(image=images, extrinsics=ctx_e, intrinsics=ctx_k, near=near_c, far=far_c)
    loss_depth = L.LossDepth(L.LossDepthCfgWrapper(L.LossDepthCfg(0.25, 12.0, True)))
    batch = {"target": {"near": near_t, "far": far_t, "image": target}}
    params = list(enc.parameters()) + list(head.parameters())

    def step():
        torch.manual_seed(7)                 # the depth predictor samples its depth buckets at random in training
        x = feats.clone().requires_grad_(True)
        for p in params:
            p.grad = None
        f, _ = enc(x, ctx_e, ctx_k, near_c, far_c)
        gs = head(f, context, global_step=0)
        out, sse, _ = dec.forward_mse(gs, tgt_e, tgt_k, near_t, far_t, (HW, HW), target, depth_mode="depth")
        loss = L.mse_from_sse(sse, (HW, HW)) + loss_depth(out, batch) + \
            (1 - L.ssim(target.flatten(0, 1), out.color.flatten(0, 1))).mean()
        loss.backward()
        return [loss.detach(), x.grad] + [p.grad for p in params]

    a, b = step(), step()
    assert torch.isfinite(a[0]) and a[1].abs().sum() > 0
    assert sum(p is not None for p in a[2:]) > 10
    for i, (u, v) in enumerate(zip(a, b)):
        assert (u is None and v is None) or torch.equal(u, v), i


# ------------------------------------------------------------------ 6. flag off
def test_flag_off_calls_the_atomic_entry_point(monkeypatch):
    from pixelsplat_b200 import _lib
    calls = []
    for name in ("ps_epipolar_attention_backward", "ps_epipolar_attention_backward_deterministic"):
        fn = getattr(_lib.lib, name)
        monkeypatch.setattr(_lib.lib, name, lambda *a, _fn=fn, _n=name: (calls.append(_n), _fn(*a))[1])
    geom, heads, x = _case(*CASES["h4-s7-pe0-v3-6x10"])
    flag = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(False)
        _backward(geom, heads, x)
        assert calls == ["ps_epipolar_attention_backward"]
        torch.use_deterministic_algorithms(True)
        _backward(geom, heads, x)
        assert calls == ["ps_epipolar_attention_backward", "ps_epipolar_attention_backward_deterministic"]
    finally:
        torch.use_deterministic_algorithms(flag)
