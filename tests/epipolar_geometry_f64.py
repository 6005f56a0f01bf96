"""A plain float64 restatement of one `ps_epipolar_geometry` call (include/pixelsplat_b200.h), the yardstick of
k_epipolar_geometry (csrc/epipolar_geometry.cu), written from the reference's math (EpipolarSampler.forward,
project_rays, get_depth, depth_to_relative_disparity), in numpy.

For batch b, view v (the query camera), other view ov (camera o = ov < v ? ov : ov + 1) and ray r of the h x w grid:
  xy         = ((col + 0.5) / w, (row + 0.5) / h)
  d_c        = K_v^-1 (x, y, 1) / |K_v^-1 (x, y, 1)|,   d = R_v d_c,  origin = t_v            (get_world_rays)
  o', d'     = E_o^-1 applied to (origin, 1) and (d, 0)                                      (camera o's space)
  frame hits the four lines x = 0, x = 1, y = 0, y = 1 of camera o's image; a hit is valid when its xy is within
             [-1e-6, 1 + 1e-6], its z > -1e-6 and its t > -1e-6; the first minimum / maximum of t over the valid
             ones (invalid ones ranked +inf / -inf)
  near / far the projection of o' + t d' at t = near_v / far_v: p / (p_z + eps32), nan_to_num(+-1e8), then K_o; its
             validity is the same rule
  lo, hi     near (far) projection if valid, else the frame minimum (maximum); overlap = lo.valid & hi.valid
  segment    nan_to_num(lo.xy, hi.xy) (every non-finite to 0), times the overlap; t_range = (lo.t, hi.t)
  sample s   xy_s = x0 + u (x1 - x0), u = (s + 0.5) / S
  depth      closest point p of the query ray and camera o's world ray through xy_s (closed form: the midpoint of the
             common perpendicular); rays with d . d2 > 1 - 1e-5 are parallel and p = (1e10, 1e10, 1e10); depth = |p -
             origin| clipped to [near_v, far_v]
  rel_disparity = 1 - (1 / (depth + eps) - 1 / (far_v + eps)) / (1 / (near_v + eps) - 1 / (far_v + eps) + eps),
             eps = 1e-10

Two modes:
  "reference"  every step in float64, which is what the reference computes on float64 cameras
  "kernel"     the same, except the sample position is formed as the reference forms it in float32 (the dtype of the
               kernel's cameras): u = f32((s + 0.5) / S), xy_s = f32(x0 + f32(u * f32(x1 - x0))) on the float32 segment
               ends.  Everything else stays float64, as in the kernel.

`geometry` also returns, per ray and per sample, the distance of every discrete decision from its threshold
("margins"), each divided by the size of the quantity it compares, so that `flags` can excuse exactly the elements
that sit on a decision boundary, where float64 rounding in another order could take the other branch:
  ray     every in-bounds comparison (x, y against -1e-6 and 1 + 1e-6), z > -1e-6 and t > -1e-6 of every projection
          that can become an end (the near / far projection always, the frame hits on a side whose near / far
          projection is invalid or itself flagged), and the gap between the first and second smallest (largest) valid
          frame-hit t on such a side
  sample  the parallel threshold |c - (1 - 1e-5)|, anti-parallel rays 1 + c (where the closest point is
          ill-conditioned), and the near and far clips |depth - near| / near, |depth - far| / far
"""
from __future__ import annotations

import numpy as np

EPS_BOUNDS = 1e-6
EPS32 = float(np.finfo(np.float32).eps)
PARALLEL = 1.0 - 1e-5
EPS_DISP = 1e-10


def _nan_to_num(x, pinf, ninf):
    return np.nan_to_num(x, nan=0.0, posinf=pinf, neginf=ninf)


def _rel(m, scale):
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.abs(m) / np.maximum(np.abs(scale), 1.0)
    return np.where(np.isnan(r), np.inf, r)          # a NaN compares false on every path: no boundary to sit on


def _valid_margins(x, y, z, t, z_scale):
    """(valid, margin): the in-bounds / in-front / positive-t rule and its least relative distance to a threshold."""
    with np.errstate(invalid="ignore"):
        valid = ((x >= -EPS_BOUNDS) & (y >= -EPS_BOUNDS) & (x <= 1 + EPS_BOUNDS) & (y <= 1 + EPS_BOUNDS)
                 & (z > -EPS_BOUNDS) & (t > -EPS_BOUNDS))
    m = np.minimum.reduce([_rel(x + EPS_BOUNDS, 1.0), _rel(y + EPS_BOUNDS, 1.0), _rel(1 + EPS_BOUNDS - x, 1.0),
                           _rel(1 + EPS_BOUNDS - y, 1.0), _rel(z + EPS_BOUNDS, z_scale), _rel(t + EPS_BOUNDS, t)])
    return valid, m


def _frame_hit(K, o, d, dim, value):
    od = 1 - dim
    fs, fo, cs, co = K[..., dim, dim], K[..., od, od], K[..., dim, 2], K[..., od, 2]
    os_, oo, ds, do, oz, dz = o[..., dim], o[..., od], d[..., dim], d[..., od], o[..., 2], d[..., 2]
    c = (value - cs) / fs
    with np.errstate(invalid="ignore", divide="ignore"):
        t = (c * oz - os_) / (ds - c * dz)
        other = co + fo * (oo * (c * dz - ds) + do * (os_ - c * oz)) / (dz * os_ - ds * oz)
        z = oz + t * dz
        same = np.full(other.shape, value)
        x, y = (same, other) if dim == 0 else (other, same)
        valid, _ = _valid_margins(x, y, z, t, np.abs(oz) + np.abs(t * dz))
        mid = np.full(other.shape, 0.5)            # the hit's own coordinate is the frame line exactly: no boundary
        _, m = _valid_margins(*((mid, other) if dim == 0 else (other, mid)), z, t, np.abs(oz) + np.abs(t * dz))
    return t, x, y, valid, m


def _point_proj(K, o, d, t):
    p = o + t[..., None] * d
    with np.errstate(invalid="ignore", divide="ignore"):
        q = _nan_to_num(p / (p[..., 2:] + EPS32), 1e8, -1e8)
    xy = np.einsum("...ij,...j->...i", K[..., :2, :], q)
    valid, m = _valid_margins(xy[..., 0], xy[..., 1], p[..., 2], t, np.abs(o[..., 2]) + np.abs(t * d[..., 2]))
    return xy[..., 0], xy[..., 1], valid, m


def other_view(v: int, ov: int) -> int:
    return ov if ov < v else ov + 1


def geometry(extrinsics, intrinsics, near, far, grid, samples: int, mode: str = "kernel") -> dict:
    """extrinsics [b, v, 4, 4] camera-to-world, intrinsics [b, v, 3, 3] (normalised), near / far [b, v], any float
    dtype (widened to float64).  Returns numpy arrays: segments [b, v, ov, r, 4], valid [b, v, ov, r] bool,
    t_range [b, v, ov, r, 2], rel_disparity [b, v, ov, r, s], ray_margin [b, v, ov, r] and sample_margin
    [b, v, ov, r, s] (the least relative distance to a decision; the sample margin includes its ray's), plus each
    sample decision's own margin under "sample_margins"."""
    assert mode in ("reference", "kernel")
    f64 = lambda a: np.asarray(a.detach().cpu() if hasattr(a, "detach") else a, dtype=np.float64)
    E, K, near, far = f64(extrinsics), f64(intrinsics), f64(near), f64(far)
    b, v = E.shape[:2]
    h, w = grid
    S = samples
    ov_idx = np.array([[other_view(vi, o) for o in range(v - 1)] for vi in range(v)], dtype=np.int64).reshape(v, v - 1)
    Eo, Ko = E[:, ov_idx], K[:, ov_idx]                              # [b, v, ov, ...]
    nearv, farv = near[:, :, None, None], far[:, :, None, None]      # the query camera's planes, [b, v, 1, 1]

    # --- world rays of the query views at the cell centres
    cols, rows = np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64)
    gx, gy = np.meshgrid((cols + 0.5) / w, (rows + 0.5) / h, indexing="xy")
    pix = np.stack([gx.reshape(-1), gy.reshape(-1), np.ones(h * w)], -1)            # [r, 3]
    dc = np.einsum("bvij,rj->bvri", np.linalg.inv(K), pix)
    dc = dc / np.linalg.norm(dc, axis=-1, keepdims=True)
    dw = np.einsum("bvij,bvrj->bvri", E[..., :3, :3], dc)                            # [b, v, r, 3]
    ow = E[..., :3, 3]                                                               # [b, v, 3]

    # --- into the other cameras' space
    w2c = np.linalg.inv(Eo)                                                          # [b, v, ov, 4, 4]
    oc = np.einsum("bvoij,bvj->bvoi", w2c[..., :3, :3], ow) + w2c[..., :3, 3]         # [b, v, ov, 3]
    oc = np.broadcast_to(oc[:, :, :, None], (b, v, v - 1, h * w, 3))
    dcam = np.einsum("bvoij,bvrj->bvori", w2c[..., :3, :3], dw)                      # [b, v, ov, r, 3]
    Kb = Ko[:, :, :, None]

    hits = [_frame_hit(Kb, oc, dcam, dim, val) for dim, val in ((0, 0.0), (0, 1.0), (1, 0.0), (1, 1.0))]
    ht = np.stack([hh[0] for hh in hits]); hx = np.stack([hh[1] for hh in hits]); hy = np.stack([hh[2] for hh in hits])
    hv = np.stack([hh[3] for hh in hits]); hm = np.stack([hh[4] for hh in hits])
    tlo, thi = np.where(hv, ht, np.inf), np.where(hv, ht, -np.inf)
    imin, imax = np.argmin(tlo, 0), np.argmax(thi, 0)                               # first minimum / maximum
    take = lambda a, i: np.take_along_axis(a, i[None], 0)[0]
    tmin, tmax = take(tlo, imin), take(thi, imax)

    tn = np.broadcast_to(nearv, tmin.shape)
    tf = np.broadcast_to(farv, tmin.shape)
    nx, ny, nvalid, nm = _point_proj(Kb, oc, dcam, tn)
    fx, fy, fvalid, fm = _point_proj(Kb, oc, dcam, tf)

    lo_t = np.where(nvalid, tn, tmin)
    lo_x, lo_y = np.where(nvalid, nx, take(hx, imin)), np.where(nvalid, ny, take(hy, imin))
    lo_v = np.where(nvalid, True, take(hv, imin))
    hi_t = np.where(fvalid, tf, tmax)
    hi_x, hi_y = np.where(fvalid, fx, take(hx, imax)), np.where(fvalid, fy, take(hy, imax))
    hi_v = np.where(fvalid, True, take(hv, imax))
    overlaps = lo_v & hi_v
    m = overlaps.astype(np.float64)
    x0, y0 = _nan_to_num(lo_x, 0.0, 0.0) * m, _nan_to_num(lo_y, 0.0, 0.0) * m
    x1, y1 = _nan_to_num(hi_x, 0.0, 0.0) * m, _nan_to_num(hi_y, 0.0, 0.0) * m

    # --- decision margins of the ray
    TAU_SIDE = 1e-6        # a near / far projection this close to its rule may go either way: its side's hits count
    frame_m = hm.min(0)
    with np.errstate(invalid="ignore"):                 # inf - inf where fewer than two hits are valid: no tie
        srt = np.sort(tlo, 0)
        gap_lo = _rel(srt[1] - srt[0], srt[0])
        srt = np.sort(thi, 0)
        gap_hi = _rel(srt[-1] - srt[-2], srt[-1])
    lo_side = np.where(~nvalid | (nm < TAU_SIDE), np.minimum(frame_m, gap_lo), np.inf)
    hi_side = np.where(~fvalid | (fm < TAU_SIDE), np.minimum(frame_m, gap_hi), np.inf)
    ray_margin = np.minimum.reduce([nm, fm, lo_side, hi_side])

    # --- samples
    if mode == "reference":
        u = (np.arange(S, dtype=np.float64) + 0.5) / S
        sx = x0[..., None] + u * (x1 - x0)[..., None]
        sy = y0[..., None] + u * (y1 - y0)[..., None]
    else:
        u = ((np.arange(S, dtype=np.float64) + 0.5) / S).astype(np.float32)
        f32 = lambda a: a.astype(np.float32)
        sx = (f32(x0)[..., None] + u * (f32(x1) - f32(x0))[..., None]).astype(np.float64)
        sy = (f32(y0)[..., None] + u * (f32(y1) - f32(y0))[..., None]).astype(np.float64)
    pix2 = np.stack([sx, sy, np.ones_like(sx)], -1)                                   # [b, v, ov, r, s, 3]
    d2c = np.einsum("bvoij,bvorsj->bvorsi", np.linalg.inv(Ko), pix2)
    d2c = d2c / np.linalg.norm(d2c, axis=-1, keepdims=True)
    d2 = np.einsum("bvoij,bvorsj->bvorsi", Eo[..., :3, :3], d2c)
    o2 = Eo[..., :3, 3][:, :, :, None, None]                                         # [b, v, ov, 1, 1, 3]
    o1 = ow[:, :, None, None, None]
    d1 = dw[:, :, None, :, None]
    c = (d1 * d2).sum(-1)
    parallel = c > PARALLEL
    wv = o2 - o1
    a = (wv * d1).sum(-1)
    bb = (wv * d2).sum(-1)
    with np.errstate(invalid="ignore", divide="ignore"):
        den = 1.0 - c * c
        t = (a - bb * c) / den
        sp = (a * c - bb) / den
        q = 0.5 * (o1 + t[..., None] * d1 + o2 + sp[..., None] * d2) - o1
    depth = np.linalg.norm(q, axis=-1)
    depth_par = np.linalg.norm(1e10 - o1, axis=-1)
    depth = np.where(parallel, np.broadcast_to(depth_par, depth.shape), depth)
    nears, fars = nearv[..., None], farv[..., None]
    clipped = np.minimum(np.maximum(depth, nears), fars)
    disp_near, disp_far = 1.0 / (nears + EPS_DISP), 1.0 / (fars + EPS_DISP)
    rd = 1.0 - (1.0 / (clipped + EPS_DISP) - disp_far) / (disp_near - disp_far + EPS_DISP)

    sample_margins = dict(parallel=np.abs(c - PARALLEL), antiparallel=np.where(parallel, np.inf, 1.0 + c),
                          near_clip=_rel(depth - nears, nears), far_clip=_rel(depth - fars, fars))
    sample_margin = np.minimum.reduce([*sample_margins.values(), np.broadcast_to(ray_margin[..., None], rd.shape)])
    return dict(segments=np.stack([x0, y0, x1, y1], -1), valid=overlaps, t_range=np.stack([lo_t, hi_t], -1),
                rel_disparity=rd, xy_sample=np.stack([sx, sy], -1), depth=depth, ray_margin=ray_margin,
                sample_margin=sample_margin, sample_margins=sample_margins)


def flags(g: dict, tau_ray: float, tau_parallel: float, tau_antiparallel: float, tau_clip: float):
    """(ray flags, sample flags): the elements within the given relative distance of a decision.  A flagged ray flags
    all its samples; clips are continuous, so tau_clip only matters to a bit-identity count."""
    ray = g["ray_margin"] < tau_ray
    m = g["sample_margins"]
    smp = ((m["parallel"] < tau_parallel) | (m["antiparallel"] < tau_antiparallel)
           | (m["near_clip"] < tau_clip) | (m["far_clip"] < tau_clip) | ray[..., None])
    return ray, smp
