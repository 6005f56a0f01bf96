"""A torch float64 restatement of 3DGS's adaptive density control on PLY vertex records (csrc/ply_densify.cu,
pixelsplat_b200.ply_refine): the statistics, clone / split / prune in 3DGS's output order, and the opacity reset.

Decisions follow the kernels' precision: the mean gradient norm g = accum / count and its comparison with the
threshold in float32 (as 3DGS compares its float32 norms with a Python float), the scale and opacity tests in
float64.  Split copies are formed in float64 and rounded once to float32."""
from __future__ import annotations

import math

import torch

LOG_SPLIT = math.log(1.6)          # the copies' scale is the original's / (0.8 N), N = 2
OPACITY_RESET_LOGIT = math.log(0.01 / 0.99)


def columns(names) -> dict:
    col = {k: i for i, k in enumerate(names)}
    return {"xyz": [col[k] for k in "xyz"], "opacity": col["opacity"],
            "scale": [col[f"scale_{k}"] for k in range(3)], "rot": [col[f"rot_{k}"] for k in range(4)]}


def stats_f64(d_means2d: torch.Tensor, radii: torch.Tensor, accum: torch.Tensor, count: torch.Tensor):
    """(accum + sum over views with radii > 0 of |d_means2d[v, :, :2]| in float64, count + the number of those
    views)."""
    on = radii > 0
    norms = d_means2d[..., :2].double().norm(dim=-1)
    return accum.double() + torch.where(on, norms, torch.zeros_like(norms)).sum(0), count + on.sum(0).to(count.dtype)


def rotation_f64(q: torch.Tensor) -> torch.Tensor:
    """[n, 4] wxyz -> R(q^) [n, 3, 3] in float64; a zero quaternion is the identity."""
    q = q.double()
    n2 = (q * q).sum(-1, keepdim=True)
    ident = torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=torch.float64).expand_as(q)
    q = torch.where(n2 > 0, q / torch.sqrt(torch.where(n2 > 0, n2, torch.ones_like(n2))), ident)
    w, x, y, z = q.unbind(-1)
    return torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                        torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def mean_grad(accum: torch.Tensor, count: torch.Tensor) -> torch.Tensor:
    """g = accum / count in float32, 0 where count = 0."""
    return torch.where(count > 0, accum.float() / count.clamp(min=1).float(), torch.zeros_like(accum.float()))


def prunes(opacity: torch.Tensor, log_scales: torch.Tensor, cfg, prune_world: bool) -> torch.Tensor:
    transparent = 1.0 / (1.0 + torch.exp(-opacity.double())) < cfg.min_opacity
    if not prune_world:
        return transparent
    return transparent | (log_scales.double().exp().amax(-1) > 0.1 * cfg.extent)


def split_copies(records: torch.Tensor, names, eps: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """Both copies of every record (float32 [n, P] each): p' = p + R(q^) (exp(l) * eps[k]), l' = l - log(1.6), in
    float64 rounded once; every other column copied."""
    c = columns(names)
    rot = rotation_f64(records[:, c["rot"]])
    s = records[:, c["scale"]].double().exp()
    out = []
    for k in range(2):
        copy = records.clone()
        se = s * eps[k].double()
        copy[:, c["xyz"]] = (records[:, c["xyz"]].double() + (rot * se[:, None, :]).sum(-1)).float()
        copy[:, c["scale"]] = (records[:, c["scale"]].double() - LOG_SPLIT).float()
        out.append(copy)
    return out[0], out[1]


def flags(records: torch.Tensor, accum: torch.Tensor, count: torch.Tensor, names, cfg, prune_world: bool):
    """(keep, clone, split) boolean [n]: the original kept, a kept clone, two kept split copies."""
    c = columns(names)
    l = records[:, c["scale"]]
    o = records[:, c["opacity"]]
    selected = mean_grad(accum, count) >= torch.tensor(cfg.grad_threshold, dtype=torch.float32)
    big = l.double().exp().amax(-1) > cfg.percent_dense * cfg.extent
    pruned = prunes(o, l, cfg, prune_world)
    l2 = (l.double() - LOG_SPLIT).float()
    return ~(selected & big) & ~pruned, selected & ~big & ~pruned, selected & big & ~prunes(o, l2, cfg, prune_world)


def densify_f64(records, exp_avg, exp_avg_sq, accum, count, names, cfg, prune_world: bool, eps):
    """-> (records, exp_avg, exp_avg_sq) of the densified set: kept originals, kept clones, first split copies,
    second split copies, each in input order; moments copied for kept originals and zero for new rows."""
    keep, clone, split = flags(records, accum, count, names, cfg, prune_world)
    first, second = split_copies(records, names, eps)
    rec = torch.cat([records[keep], records[clone], first[split], second[split]])
    new = int(clone.sum()) + 2 * int(split.sum())
    zeros = torch.zeros((new, records.shape[1]), dtype=records.dtype)
    return rec, torch.cat([exp_avg[keep], zeros]), torch.cat([exp_avg_sq[keep], zeros])


def reset_opacity_f64(records, exp_avg, exp_avg_sq, names):
    """o = min(o, logit(0.01)) (the logit rounded to float32) and the opacity column's moments zeroed."""
    c = columns(names)["opacity"]
    rec, m, v = records.clone(), exp_avg.clone(), exp_avg_sq.clone()
    rec[:, c] = torch.minimum(rec[:, c], torch.tensor(OPACITY_RESET_LOGIT, dtype=torch.float32))
    m[:, c] = 0.0
    v[:, c] = 0.0
    return rec, m, v
