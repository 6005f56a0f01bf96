"""A plain float64 restatement of one `ps_gaussian_adapter_forward` / `ps_gaussian_adapter_backward` call
(include/pixelsplat_b200.h), the yardstick of the fused adapter kernels (csrc/gaussian_adapter.cu), and the
per-entry bars they are held to.

For view v (camera-to-world E = [C | o], intrinsics K), ray r (coordinates (x, y); raw row = scale logits s [3],
quaternion qr [4] xyzw, sh [3, n]) and sample j (depth t):
  sigma      = scale_min + (scale_max - scale_min) sigmoid(s)
  mult       = 0.1 sum(K[:2, :2]^-1 (1 / w, 1 / h))    (1 / w and 1 / h rounded to float32, as the kernel and the
                                                        reference's get_scale_multiplier take them)
  scales     = sigma t mult
  q          = qr / (|qr| + eps),  R = quaternion_to_matrix(q) with 2 / (q.q + eps)
  covariance = (C R) diag(scales^2) (C R)^T
  d          = K^-1 (x, y, 1),  means = o + t C d / |d|
  harmonics  = D (mask * sh[c]) per colour channel c, the same for every sample of the ray
  rotations  = q, one per ray
D is the block-diagonal SH rotation exactly as the kernel received it (float32 values, widened), so the adapter is
compared in isolation from k_sh_rotation.  The gradients are autograd of <outputs, cotangents>.  Everything is dense
torch arithmetic on the inputs' device.

Bars (`ratios`, `check`): every entry of every output and gradient is held, |got - ref| <= BAR[kind] * scale, where
the scale is the entry's own (returned by `forward_backward` under "scale"):
  means              |o| + t of the Gaussian                    (a translation error and a depth error alike)
  covariances        the Gaussian's largest float64 variance    (its largest |entry|: sizes span (far / near)^2
                                                                across Gaussians; 4e-6 of it stays under today's
                                                                5e-6 of the whole tensor's largest entry)
  scales             |ref|
  rotations          1                                          (unit quaternions)
  harmonics          2-norm of the (Gaussian, channel, degree) block of the float64 result (a rotation keeps it)
  d_raw sh part      mask_l ||sum_samples |d_harm| block|| per (ray, channel, degree): the rotation keeps the norm,
                     and the kernel's float32 sum over the samples rounds with the size of its terms, not of the sum
                     (random per-sample cotangents cancel: a degree-0 sum can be 1e-3 of its terms)
  d_raw[0:7], d_depths, d_coordinates
                     |ref| + GRAD_MIX * S, S = the component's largest |ref| over the call.  These are sums whose
                     terms cancel (over the samples, and the projections of the normalisations); S stands for the
                     terms' size.  Over the call rather than the view, because a view may hold one ray.
A failure names view, ray, sample, component and degree block, and the ray's (blockIdx.x, warp, lane) in the
kernels' 128-ray blocks.
"""
from __future__ import annotations

import math

import numpy as np
import torch

F64 = torch.float64
RAYS_PER_BLOCK = 128

# Measured on an NVIDIA H100 80GB HBM3 (see DESIGN.md section 9 "Parity" and tests/test_adapter_sweep_gpu.py for
# the worst case of each); each bar is at least 3x the worst measured error-to-scale ratio.
BAR = dict(means=1e-6, covariances=4e-6, scales=1.2e-6, rotations=5e-7, harmonics=8e-7, d_raw_sh=7e-7,
           d_raw=1e-5, d_depths=6e-6, d_coordinates=6e-6)
GRAD_MIX = 0.1          # the absolute part of the mixed gradient bars: GRAD_MIX * BAR * (the view's largest |ref|)

OUTPUTS = ("means", "covariances", "harmonics", "scales", "rotations")
GRADIENTS = ("d_coordinates", "d_depths", "d_raw")


def widen(x: float) -> float:
    """The float32 value the kernel receives for a descriptor field, as a float64."""
    return float(np.float32(x))


def sh_mask(n_sh: int) -> torch.Tensor:
    """GaussianAdapter's sh_mask (1 for degree 0, 0.1 * 0.25^l above), float32 values as float64."""
    m = torch.ones(n_sh, dtype=torch.float32)
    for l in range(1, math.isqrt(n_sh)):
        m[l * l:(l + 1) ** 2] = 0.1 * 0.25 ** l
    return m.double()


def degree_of(k: int) -> int:
    """The SH degree of coefficient k."""
    return math.isqrt(k)


def sh_degree(n_sh: int) -> int:
    """The SH degree of a basis of n_sh = (degree + 1)^2 coefficients."""
    return math.isqrt(n_sh) - 1


def quaternion_to_matrix(q: torch.Tensor, eps: float) -> torch.Tensor:
    i, j, k, r = q.unbind(-1)
    ts = 2.0 / ((q * q).sum(-1) + eps)
    o = torch.stack((1 - ts * (j * j + k * k), ts * (i * j - k * r), ts * (i * k + j * r),
                     ts * (i * j + k * r), 1 - ts * (i * i + k * k), ts * (j * k - i * r),
                     ts * (i * k - j * r), ts * (j * k + i * r), 1 - ts * (i * i + j * j)), -1)
    return o.reshape(*q.shape[:-1], 3, 3)


def forward(E, K, D, mask, coordinates, depths, raw, image_hw, scale_min, scale_max, eps) -> dict:
    """E [nv, 4, 4], K [nv, 3, 3], D [nv, n, n], mask [n], coordinates [nv, nr, 2], depths [nv, nr, ns],
    raw [nv, nr, 7 + 3 n] -> means [nv, nr, ns, 3], covariances [.., 3, 3], harmonics [.., 3, n], scales [.., 3],
    rotations [nv, nr, 4], all float64 and differentiable in coordinates, depths and raw."""
    E, K, D, mask = E.double(), K.double(), D.double(), mask.double()
    coordinates, depths, raw = coordinates.double(), depths.double(), raw.double()
    nv, nr, ns = depths.shape
    n = mask.shape[0]
    dev = raw.device
    C, o = E[:, :3, :3], E[:, :3, 3]
    s, qr, sh = raw[..., :3], raw[..., 3:7], raw[..., 7:].reshape(nv, nr, 3, n)
    sigma = scale_min + (scale_max - scale_min) * torch.sigmoid(s)
    h, w = image_hw
    px = torch.tensor([widen(1.0 / w), widen(1.0 / h)], dtype=F64, device=dev)
    mult = 0.1 * (torch.linalg.inv(K[:, :2, :2]) @ px).sum(-1)                       # [nv]
    scales = sigma[:, :, None, :] * depths[..., None] * mult[:, None, None, None]      # [nv, nr, ns, 3]
    q = qr / (torch.linalg.vector_norm(qr, dim=-1, keepdim=True) + eps)
    A = C[:, None] @ quaternion_to_matrix(q, eps)                                      # [nv, nr, 3, 3]
    cov = torch.einsum("vrik,vrsk,vrjk->vrsij", A, scales * scales, A)
    xy1 = torch.cat([coordinates, torch.ones_like(coordinates[..., :1])], -1)
    d = torch.einsum("vij,vrj->vri", torch.linalg.inv(K), xy1)
    d = d / torch.linalg.vector_norm(d, dim=-1, keepdim=True)
    dw = torch.einsum("vij,vrj->vri", C, d)
    means = o[:, None, None, :] + dw[:, :, None, :] * depths[..., None]
    harm = torch.einsum("vij,vrcj->vrci", D, sh * mask)
    return dict(means=means, covariances=cov, harmonics=harm[:, :, None].expand(nv, nr, ns, 3, n), scales=scales,
                rotations=q)


def _block_norms(x: torch.Tensor) -> torch.Tensor:
    """x [..., n] -> [..., n]: each entry replaced by the 2-norm of its degree block."""
    out = torch.empty_like(x)
    for l in range(math.isqrt(x.shape[-1])):
        s = slice(l * l, (l + 1) ** 2)
        out[..., s] = torch.linalg.vector_norm(x[..., s], dim=-1, keepdim=True)
    return out


def _mixed(ref: torch.Tensor, dims) -> torch.Tensor:
    return ref.abs() + GRAD_MIX * ref.abs().amax(dim=dims, keepdim=True)


def forward_backward(E, K, D, mask, coordinates, depths, raw, image_hw, scale_min, scale_max, eps,
                     cot: dict) -> dict:
    """forward() plus d_coordinates, d_depths and d_raw for the cotangents `cot` (keys d_means, d_cov, d_harm,
    d_scales, d_rot; a missing or None one is zero), every result detached float64, and "scale": the scale of each
    entry's bar (module docstring)."""
    leaves = [t.detach().double().requires_grad_(True) for t in (coordinates, depths, raw)]
    out = forward(E, K, D, mask, *leaves, image_hw, scale_min, scale_max, eps)
    names = dict(d_means="means", d_cov="covariances", d_harm="harmonics", d_scales="scales", d_rot="rotations")
    loss = sum((out[o] * cot[c].double()).sum() for c, o in names.items() if cot.get(c) is not None)
    g = torch.autograd.grad(loss, leaves, allow_unused=True)
    res = {k: v.detach() for k, v in out.items()}
    res.update({k: (torch.zeros_like(l) if x is None else x.detach()) for k, x, l in zip(GRADIENTS, g, leaves)})
    n = res["harmonics"].shape[-1]
    mask = mask.double().to(res["means"].device)
    o_norm = torch.linalg.vector_norm(E.double()[:, :3, 3], dim=-1).to(res["means"].device)
    sc = dict(means=(o_norm[:, None, None, None] + depths.double()[..., None]).expand_as(res["means"]),
              covariances=res["covariances"].diagonal(dim1=-2, dim2=-1).amax(-1)[..., None, None]
              .expand_as(res["covariances"]),
              scales=res["scales"].abs(), rotations=torch.ones_like(res["rotations"]),
              harmonics=_block_norms(res["harmonics"]),
              d_depths=_mixed(res["d_depths"], (0, 1, 2)), d_coordinates=_mixed(res["d_coordinates"], (0, 1)))
    dr = torch.empty_like(res["d_raw"])
    dr[..., :7] = _mixed(res["d_raw"][..., :7], (0, 1))
    dh = cot.get("d_harm")
    dh = torch.zeros_like(res["harmonics"]) if dh is None else dh.double()
    dr[..., 7:] = (mask * _block_norms(dh.abs().sum(2))).reshape(dr.shape[0], dr.shape[1], 3 * n)
    sc["d_raw"] = dr
    res["scale"] = sc
    return res


def allowed(key: str, scale: torch.Tensor) -> torch.Tensor:
    """|got - ref| may reach this: the bar of `key` times the entries' scales (d_raw: two bars, head and sh part)."""
    if key != "d_raw":
        return BAR[key] * scale
    a = BAR["d_raw"] * scale
    a[..., 7:] = BAR["d_raw_sh"] * scale[..., 7:]
    return a


def describe(key: str, idx, n_sh: int) -> str:
    """Where an entry sits: view, ray, sample, component, degree block, and the ray's kernel coordinates."""
    idx = [int(i) for i in idx]
    v, r, rest = idx[0], idx[1], idx[2:]
    parts = [f"view {v}", f"ray {r}"]
    if key in ("means", "scales", "covariances", "harmonics", "d_depths"):
        parts.append(f"sample {rest[0]}")
        rest = rest[1:]
    if key == "covariances":
        parts.append(f"component ({rest[0]}, {rest[1]})")
    elif key == "harmonics":
        parts.append(f"channel {rest[0]} coefficient {rest[1]} (degree {degree_of(rest[1])})")
    elif key == "d_raw":
        k = rest[0]
        if k < 3:
            parts.append(f"scale logit {k}")
        elif k < 7:
            parts.append(f"quaternion component {k - 3}")
        else:
            c, j = divmod(k - 7, n_sh)
            parts.append(f"sh channel {c} coefficient {j} (degree {degree_of(j)})")
    elif rest:
        parts.append(f"component {rest[0]}")
    parts.append(f"(blockIdx.x {r // RAYS_PER_BLOCK}, warp {(r % RAYS_PER_BLOCK) // 32}, lane {r % 32})")
    return " ".join(parts)


def ratios(got: dict, ref: dict, keys=None) -> dict:
    """{bar: (worst |got - ref| / allowed over every entry, where it is, got, ref)}, d_raw reported as its two bars
    d_raw (components 0-6) and d_raw_sh; a NaN counts as infinitely bad."""
    out = {}
    n_sh = ref["harmonics"].shape[-1]
    for k in keys if keys is not None else OUTPUTS + GRADIENTS:
        g, r = got[k].detach().to(ref[k].device).double(), ref[k]
        assert g.shape == r.shape, (k, tuple(g.shape), tuple(r.shape))
        q = torch.nan_to_num((g - r).abs() / allowed(k, ref["scale"][k]), nan=math.inf, posinf=math.inf)
        q = torch.where((g == r), torch.zeros_like(q), q)          # exact zeros against a zero scale
        parts = [(k, 0, q)] if k != "d_raw" else [("d_raw", 0, q[..., :7]), ("d_raw_sh", 7, q[..., 7:])]
        for name, off, qp in parts:
            i = int(qp.argmax())
            idx = list(np.unravel_index(i, tuple(qp.shape)))
            idx[-1] += off
            flat = int(np.ravel_multi_index(tuple(idx), tuple(q.shape)))
            out[name] = (float(qp.reshape(-1)[i]), describe(k, idx, n_sh), float(g.reshape(-1)[flat]),
                         float(r.reshape(-1)[flat]))
    return out


def check(got: dict, ref: dict, tag: str = "", keys=None) -> dict:
    """Every entry of every key within its bar; returns {key: worst ratio}."""
    rep = ratios(got, ref, keys)
    print("ADAPTER_RATIOS", tag, " ".join(f"{k}={v[0]:.3f}" for k, v in rep.items()))
    for k, (q, where, g, r) in rep.items():
        assert q <= 1.0, f"{tag}: {k} at {where} is {q:.2f}x its bar: got {g:.9e} ref {r:.9e}"
    return {k: v[0] for k, v in rep.items()}
