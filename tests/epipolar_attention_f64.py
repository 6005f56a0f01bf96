"""A plain float64 restatement of one `_EpipolarAttentionFn` call (pixelsplat_b200/encoder/attention_fused.py), the
yardstick of the fused epipolar attention kernels (csrc/epipolar_attention.cu, include/pixelsplat_b200.h).

For query n = (b, v, r) with r = row * w + col, head h, other view ov (the view o = ov if ov < v else ov + 1) and
sample s of that ray's segment (x0, y0, x1, y1):
  xy_s   = (x0, y0) + u_s ((x1, y1) - (x0, y0)),   u_s = (s + 0.5) / S
  f_s    = bilinear(feat[b, o], xy_s) * valid      grid_sample(align_corners=False, padding_mode="zeros")
  PE_s   = [sin(w_k rd_s), cos(w_k rd_s)]_k,       w_k = float32(2 pi) 2^k   (layout "(d f p)")
  score  = qt_h . f_s + pq_h . PE_s (+ bias_h,ov),  a = soft-max over all (ov, s)
  z_h = sum a f_s,  e_h = sum a PE_s,  mass_h,ov = sum_s a,  lse_h = log sum exp score.
The gradients are autograd of <z, dz> + <e, de> + <mass, dmass>.

Everything is dense torch arithmetic (the bilinear taps become a weight matrix over the map's texels), so it runs on
any device, for any channel count, and its backward has no scatter: it works under
torch.use_deterministic_algorithms(True) as well.
"""
from __future__ import annotations

import math

import numpy as np
import torch

TWO_PI_F32 = float(np.float32(2 * math.pi))     # the reference's frequency buffer is float32(2 pi) * 2^k


def other_views(v: int) -> list[list[int]]:
    """other_views(v)[vi][ov]: the view that other view ov of view vi is."""
    return [[ov if ov < vi else ov + 1 for ov in range(v - 1)] for vi in range(v)]


def sample_positions(segments: torch.Tensor, S: int) -> torch.Tensor:
    """[..., 4] segments (xy_min, xy_max) -> [..., S, 2] normalised sample positions."""
    seg = segments.double()
    u = (torch.arange(S, dtype=torch.float64, device=seg.device) + 0.5) / S
    lo, hi = seg[..., None, :2], seg[..., None, 2:]
    return lo + u[:, None] * (hi - lo)


def bilinear_weights(xy: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """[..., 2] normalised positions -> [..., h * w] bilinear weights over the texels (zero padding: taps off the map
    get no weight)."""
    ix, iy = xy[..., 0] * w - 0.5, xy[..., 1] * h - 0.5
    x0, y0 = torch.floor(ix), torch.floor(iy)
    ax, ay = ix - x0, iy - y0
    texel = torch.arange(h * w, device=xy.device)
    out = torch.zeros((*xy.shape[:-1], h * w), dtype=torch.float64, device=xy.device)
    for dy, wy in ((0, 1 - ay), (1, ay)):
        for dx, wx in ((0, 1 - ax), (1, ax)):
            xi, yi = x0 + dx, y0 + dy
            inside = (xi >= 0) & (xi < w) & (yi >= 0) & (yi < h)
            idx = torch.where(inside, yi * w + xi, torch.full_like(xi, -1)).long()
            out = out + (wx * wy * inside)[..., None] * (idx[..., None] == texel)
    return out


def sample_features(feat_cl: torch.Tensor, segments: torch.Tensor, valid: torch.Tensor, S: int) -> torch.Tensor:
    """feat_cl [b, v, h, w, C] (channels-last), segments [b, v, ov, R, 4], valid [b, v, ov, R]
    -> [b, v, ov, R, S, C] bilinear samples times valid, differentiable in feat_cl."""
    b, v, h, w, C = feat_cl.shape
    ov, R = v - 1, h * w
    sel = torch.zeros((v, ov, v), dtype=torch.float64, device=feat_cl.device)      # one-hot view selection
    for vi, row in enumerate(other_views(v)):
        for o, src in enumerate(row):
            sel[vi, o, src] = 1.0
    maps = torch.einsum("vop,bptc->bvotc", sel, feat_cl.double().reshape(b, v, R, C))      # [b, v, ov, R, C]
    wts = bilinear_weights(sample_positions(segments, S), h, w)                           # [b, v, ov, R, S, R]
    f = torch.einsum("bvorst,bvotc->bvorsc", wts, maps)
    return f * valid.double()[..., None, None]


def positional_encoding(rd: torch.Tensor, npe: int) -> torch.Tensor:
    """[...] relative disparities -> [..., npe] = sin / cos(float32(2 pi) 2^k rd), k < npe / 2, layout "(d f p)"."""
    freq = TWO_PI_F32 * 2.0 ** torch.arange(npe // 2, dtype=torch.float64, device=rd.device)
    ph = rd.double()[..., None] * freq
    return torch.stack([torch.sin(ph), torch.cos(ph)], -1).reshape(*rd.shape, npe)


def forward(feat_cl, segments, valid, rel_disparity, qt, pq, bias, heads: int) -> dict:
    """z [N, H, C], e [N, H, npe], mass [N, H, ov], lse [N, H] in float64, differentiable in feat_cl, qt, pq, bias
    (whichever require grad).  N = b v h w queries in (b, v, row, col) order."""
    b, v, h, w, C = feat_cl.shape
    ov, R, S = v - 1, h * w, rel_disparity.shape[-1]
    n, npe = b * v * R, pq.shape[-1]
    f = sample_features(feat_cl, segments, valid, S)                                     # [b, v, ov, R, S, C]
    f = f.permute(0, 1, 3, 2, 4, 5).reshape(n, ov, S, C)
    pe = positional_encoding(rel_disparity.permute(0, 1, 3, 2, 4).reshape(n, ov, S), npe)   # [n, ov, S, npe]
    qt, pq = qt.double().reshape(n, heads, C), pq.double().reshape(n, heads, npe)
    score = torch.einsum("nhc,nosc->nhos", qt, f) + torch.einsum("nhj,nosj->nhos", pq, pe)
    if bias is not None:
        score = score + bias.double().reshape(n, heads, ov)[..., None]
    flat = score.reshape(n, heads, ov * S)
    lse = torch.logsumexp(flat, -1)
    a = torch.exp(flat - lse[..., None]).reshape(n, heads, ov, S)
    return dict(z=torch.einsum("nhos,nosc->nhc", a, f), e=torch.einsum("nhos,nosj->nhj", a, pe),
                mass=a.sum(-1), lse=lse, a=a, samples=f, pe=pe)


def forward_backward(feat_cl, segments, valid, rel_disparity, qt, pq, bias, heads: int, dz, de, dmass=None) -> dict:
    """forward() plus dqt, dpq, dbias (None without a bias) and dfeat: autograd of <z, dz> + <e, de> (+ <mass, dmass>).
    All eight results are detached float64 tensors.

    Also the cancellation scales dqt_scale, dpq_scale, dbias_scale: the score gradient is a (da - D) with
    da = dz.f + de.PE (+ dmass) and D = sum a da over the row, so dqt = sum a (da - D) f can vanish by construction
    (one other view for dbias; a row whose samples are all alike for dqt and dpq) while each term does not.  The
    scales are the same sums over a (|da| + |D|): the size of the terms a float32 evaluation rounds."""
    leaves = {k: t.detach().double().requires_grad_(True)
              for k, t in dict(qt=qt, pq=pq, bias=bias, feat=feat_cl).items() if t is not None}
    out = forward(leaves["feat"], segments, valid, rel_disparity, leaves["qt"], leaves["pq"], leaves.get("bias"), heads)
    loss = (out["z"] * dz.double()).sum() + (out["e"] * de.double()).sum()
    if dmass is not None:
        loss = loss + (out["mass"] * dmass.double()).sum()
    grads = dict(zip(leaves, torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)))
    res = {k: out[k].detach() for k in ("z", "e", "mass", "lse")}
    with torch.no_grad():
        a, f, pe = out["a"], out["samples"], out["pe"]
        da = torch.einsum("nhc,nosc->nhos", dz.double().reshape(a.shape[0], a.shape[1], -1), f) + \
            torch.einsum("nhj,nosj->nhos", de.double().reshape(a.shape[0], a.shape[1], -1), pe)
        if dmass is not None:
            da = da + dmass.double().reshape(a.shape[:3])[..., None]
        D = (a * da).sum((-1, -2), keepdim=True)
        wt = a * (da.abs() + D.abs())
        res.update(dqt_scale=torch.einsum("nhos,nosc->nhc", wt, f.abs()),
                   dpq_scale=torch.einsum("nhos,nosj->nhj", wt, pe.abs()), dbias_scale=wt.sum(-1))
    res.update(dqt=grads["qt"], dpq=grads["pq"], dbias=grads.get("bias"), dfeat=grads["feat"])
    if res["dpq"] is None:                 # pe_dim = 0: nothing depends on pq
        res["dpq"] = torch.zeros_like(leaves["pq"])
    return res
