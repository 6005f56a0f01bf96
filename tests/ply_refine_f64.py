"""A float64 restatement of ps_ply_refine_step (csrc/ply_import.cu), built on tests/ply_import_f64.py, and the same
unpack in torch ops for autograd and for a torch refinement route.

`record_grad_f64` is the step's backward in closed form (numpy, float64), with each entry's magnitude: the same
chain with every term replaced by its absolute value, which bounds the float64 rounding of the entry.  `adam_f64` is
torch.optim.Adam's update in float64, with magnitudes.  `unpack_torch` is `ply_import_f64.unpack_f64` in torch ops on
per-group tensors (any float dtype), so autograd can differentiate it."""
from __future__ import annotations

import numpy as np
import torch

from tests import ply_import_f64 as f64

GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scale", "rot")


def group_columns(names: list[str], degree: int) -> dict[str, list[int]]:
    """group -> the columns of its properties, in the group's own order (x y z; f_dc_0..2; f_rest_0..; ...)."""
    col = {n: i for i, n in enumerate(names)}
    rest = 3 * ((degree + 1) ** 2 - 1)
    return {"xyz": [col[k] for k in "xyz"], "f_dc": [col[f"f_dc_{i}"] for i in range(3)],
            "f_rest": [col[f"f_rest_{i}"] for i in range(rest)], "opacity": [col["opacity"]],
            "scale": [col[f"scale_{i}"] for i in range(3)], "rot": [col[f"rot_{i}"] for i in range(4)]}


def unpack_torch(fields: dict, degree: int, sh_coeffs: int, blocks: list, rotation=None, center=None,
                 scale: float = 1.0) -> dict:
    """fields: group -> [n, k] tensor (group_columns order) -> means, covariances, harmonics, opacities."""
    p, dt = fields["xyz"], fields["xyz"].dtype
    as_t = lambda x: torch.as_tensor(x).to(dtype=dt, device=p.device)
    m = as_t(torch.eye(3) if rotation is None else rotation)
    c = as_t(torch.zeros(3) if center is None else center)
    means = p @ m * scale + c
    q = fields["rot"]
    n2 = (q * q).sum(-1, keepdim=True)
    ident = torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=dt, device=p.device).expand_as(q)
    q = torch.where(n2 > 0, q / torch.sqrt(torch.where(n2 > 0, n2, torch.ones_like(n2))), ident)
    w, x, y, z = q.unbind(-1)
    rot = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                       torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                       torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)
    var = torch.exp(2 * fields["scale"]) * scale * scale
    b = rot.transpose(-1, -2) @ m
    cov = torch.einsum("nk,nki,nkj->nij", var, b, b)
    nc = (degree + 1) ** 2
    n = p.shape[0]
    coef = torch.cat([fields["f_dc"][:, :, None], fields["f_rest"].reshape(n, 3, nc - 1)], -1)
    parts = [coef[..., l * l:(l + 1) ** 2] @ as_t(blk).T for l, blk in enumerate(blocks[:degree + 1])]
    if sh_coeffs > nc:
        parts.append(torch.zeros(n, 3, sh_coeffs - nc, dtype=dt, device=p.device))
    harm = torch.cat(parts, -1)
    opac = torch.sigmoid(fields["opacity"][:, 0])
    return {"means": means, "covariances": cov, "harmonics": harm, "opacities": opac}


def split(records: torch.Tensor, names: list[str], degree: int) -> dict:
    return {g: records[:, cols] for g, cols in group_columns(names, degree).items()}


def record_grad_f64(records: np.ndarray, names: list[str], degree: int, blocks: list[np.ndarray], grads: dict,
                    rotation=None, center=None, scale: float = 1.0) -> tuple[np.ndarray, np.ndarray]:
    """(d_records, magnitude), float64 [n, P]: the gradient of sum(grads[k] * unpack[k]) over the records; 0 in the
    columns the unpack does not read.  `grads`: means [n, 3], covariances [n, 3, 3], harmonics [n, 3, C],
    opacities [n]."""
    return _grad(records, names, degree, blocks, grads, rotation, scale, False), \
        _grad(records, names, degree, blocks, grads, rotation, scale, True)


def _grad(records, names, degree, blocks, grads, rotation, scale, absolute):
    a = np.abs if absolute else (lambda t: t)
    sg = (lambda k: abs(k)) if absolute else (lambda k: k)
    cols = group_columns(names, degree)
    r = records.astype(np.float64)
    n = r.shape[0]
    m = a(np.eye(3) if rotation is None else np.asarray(rotation, dtype=np.float64))
    s = float(scale)
    out = np.zeros_like(r)
    gm, gc = a(grads["means"].astype(np.float64)), grads["covariances"].astype(np.float64)
    gh, go = a(grads["harmonics"].astype(np.float64)), a(grads["opacities"].astype(np.float64))
    out[:, cols["xyz"]] = s * gm @ m.T

    q = r[:, cols["rot"]]
    qn = (q * q).sum(-1)
    safe = np.where(qn > 0, qn, 1.0)
    qh = np.where(qn[:, None] > 0, q / np.sqrt(safe)[:, None], np.array([1.0, 0, 0, 0]))
    rot = f64.quat_to_matrix(q)
    var = np.exp(2 * r[:, cols["scale"]]) * s * s
    b = a(np.swapaxes(rot, -1, -2) @ (np.eye(3) if rotation is None else np.asarray(rotation, dtype=np.float64)))
    S = a(0.5 * (gc + np.swapaxes(gc, -1, -2)))
    sb = np.einsum("nij,nkj->nki", S, b)                      # S b_k
    out[:, cols["scale"]] = 2 * var * (b * sb).sum(-1)
    db = 2 * var[:, :, None] * sb                            # [n, k, j]
    dR = np.einsum("ij,nkj->nik", m, db)                     # M db^T
    w, x, y, z = a(qh).T
    R = lambda i, j: dR[:, i, j]
    dw = 2 * (sg(-1) * z * R(0, 1) + y * R(0, 2) + z * R(1, 0) + sg(-1) * x * R(1, 2) + sg(-1) * y * R(2, 0)
              + x * R(2, 1))
    dx = 2 * (y * R(0, 1) + z * R(0, 2) + y * R(1, 0) + sg(-2) * x * R(1, 1) + sg(-1) * w * R(1, 2) + z * R(2, 0)
              + w * R(2, 1) + sg(-2) * x * R(2, 2))
    dy = 2 * (sg(-2) * y * R(0, 0) + x * R(0, 1) + w * R(0, 2) + x * R(1, 0) + z * R(1, 2) + sg(-1) * w * R(2, 0)
              + z * R(2, 1) + sg(-2) * y * R(2, 2))
    dz = 2 * (sg(-2) * z * R(0, 0) + sg(-1) * w * R(0, 1) + x * R(0, 2) + w * R(1, 0) + sg(-2) * z * R(1, 1)
              + y * R(1, 2) + x * R(2, 0) + y * R(2, 1))
    dqh = np.stack([dw, dx, dy, dz], -1)
    qa = a(qh)
    dot = (qa * dqh).sum(-1, keepdims=True)
    dq = (dqh + sg(-1) * qa * dot) / np.sqrt(safe)[:, None]
    out[:, cols["rot"]] = np.where(qn[:, None] > 0, dq, 0.0)

    o = 1 / (1 + np.exp(-r[:, cols["opacity"][0]]))
    out[:, cols["opacity"][0]] = go * o * (1 - o)

    nc = (degree + 1) ** 2
    dcoef = np.zeros((n, 3, nc))
    for l, blk in enumerate(blocks[:degree + 1]):
        sl = slice(l * l, (l + 1) ** 2)
        dcoef[..., sl] = gh[..., sl] @ a(np.asarray(blk, dtype=np.float64))
    out[:, cols["f_dc"]] = dcoef[..., 0]
    out[:, cols["f_rest"]] = dcoef[..., 1:].reshape(n, -1)
    return out


def adam_f64(p, g, m, v, lr, step: int, betas=(0.9, 0.999), eps: float = 1e-15):
    """torch.optim.Adam's update in float64 (lr per entry, broadcast): -> (p, m, v) and their magnitudes."""
    p, g, m, v = (np.asarray(t, dtype=np.float64) for t in (p, g, m, v))
    b1, b2 = betas
    m2 = m + (1 - b1) * (g - m)
    v2 = b2 * v + (1 - b2) * g * g
    step_size = np.asarray(lr, dtype=np.float64) / (1 - b1 ** step)
    den = np.sqrt(v2) / np.sqrt(1 - b2 ** step) + eps
    upd = step_size * m2 / den
    # the new moment's magnitude carries into the update: a moment that nearly cancels keeps its absolute error
    m_mag = np.abs(m) + (1 - b1) * (np.abs(g) + np.abs(m))
    mags = (np.abs(p) + step_size * m_mag / den, m_mag, b2 * v + (1 - b2) * g * g)
    return (p - upd, m2, v2), mags


def adam_ratio(got, want, mag) -> np.ndarray:
    """|got - want| in float32 roundings of the entry's magnitude; an entry of magnitude 0 must be exact."""
    unit = np.finfo(np.float32).eps * mag
    err = np.abs(np.asarray(got, dtype=np.float64) - want)
    return np.where(unit > 0, err / np.where(unit > 0, unit, 1.0), np.where(err == 0, 0.0, np.inf))


class UnpackF64(torch.autograd.Function):
    """The unpack restatement with `record_grad_f64` as its backward, for gradcheck: records [n, P] float64 ->
    (means, covariances, harmonics, opacities)."""

    @staticmethod
    def forward(ctx, records, names, degree, sh_coeffs, blocks, rotation, center, scale):
        ctx.args = (records.detach().numpy(), names, degree, blocks, rotation, scale)
        with torch.no_grad():
            out = unpack_torch(split(records, names, degree), degree, sh_coeffs, blocks, rotation, center, scale)
        return out["means"], out["covariances"], out["harmonics"], out["opacities"]

    @staticmethod
    def backward(ctx, dm, dc, dh, do):
        records, names, degree, blocks, rotation, scale = ctx.args
        grads = {"means": dm.numpy(), "covariances": dc.numpy(), "harmonics": dh.numpy(), "opacities": do.numpy()}
        g, _ = record_grad_f64(records, names, degree, blocks, grads, rotation, None, scale)
        return (torch.from_numpy(g),) + (None,) * 7
