"""A plain float64 restatement of `ps_view_overlap` (include/pixelsplat_b200.h), the yardstick of k_view_overlap
(csrc/epipolar_geometry.cu), written from the reference's math (get_world_rays, project_rays with near = far = None),
in numpy.  Its frame-line intersection is tests/epipolar_geometry_f64.py's.

For the rays of frame s at the h x w pixel centres, sent into camera d:
  o, dir      camera d's view of the ray (origin t_s, direction R_s K_s^-1 (x, y, 1) normalised)
  frame       the first minimum / maximum of t over the valid hits of the four frame lines
  zero depth  at_camera = |o| < 1e-6: the projection of dir, else of o; invalid when o_z < 1e-6 and not at_camera
  infinity    the projection of dir
  overlap     (zero depth valid or frame minimum valid) and (infinity valid or frame maximum valid)

`overlap` also returns each ray's margin: the least distance of a decision that can change its overlap from that
decision's threshold, relative to the size of what it compares (the in-bounds tests 0 / 1 +- 1e-6, z > -1e-6 and
t > -1e-6 of the projections that can decide, and the gap between the two smallest / largest valid frame-hit t).
A ray whose margin is below a tolerance may take the other branch in another rounding, such as the reference's
float32.  The zero-depth mask o_z < 1e-6 and the at-camera mask |o| < 1e-6 are decided once per pair, on the
origin, whose float32 rounding error is a few ulps of the camera positions: `mask_margin` is their distance from
1e-6 over |t_src| + |t_dst| (at least 1), and MASK_TOL = 2 float32 ulps of that scale flags every ray of the pair.
"""
from __future__ import annotations

import numpy as np

from tests.epipolar_geometry_f64 import EPS32, EPS_BOUNDS, _nan_to_num, _rel

MASK_TOL = 2 * EPS32


def _rule(x, y, z, t, z_scale):
    """(valid, margin) of the in-bounds / in-front / positive-t rule.  A valid projection can turn invalid when any
    test is near its threshold (the least margin); an invalid one turns valid only when every failing test is (the
    largest failing margin).  None skips a test that is exact (a frame hit's own coordinate, t = 0 or inf)."""
    tests = [(x, 1.0, False), (y, 1.0, False), (z, z_scale, True), (t, t, True)]
    ok, margins = [], []
    with np.errstate(invalid="ignore"):
        for v, scale, strict in tests:
            if v is None:
                continue
            for dist in ((v + EPS_BOUNDS,) if strict else (v + EPS_BOUNDS, 1 + EPS_BOUNDS - v)):
                ok.append(dist > 0 if strict else dist >= 0)
                margins.append(_rel(dist, scale))
    ok, margins = np.stack(ok), np.stack(margins)
    valid = ok.all(0)
    return valid, np.where(valid, margins.min(0), np.where(ok, 0.0, margins).max(0))


def _frame_hit(K, o, d, dim, value):
    od = 1 - dim
    fs, fo, cs, co = K[dim, dim], K[od, od], K[dim, 2], K[od, 2]
    os_, oo, ds, do, oz, dz = o[..., dim], o[..., od], d[..., dim], d[..., od], o[..., 2], d[..., 2]
    c = (value - cs) / fs
    with np.errstate(invalid="ignore", divide="ignore"):
        t = (c * oz - os_) / (ds - c * dz)
        other = co + fo * (oo * (c * dz - ds) + do * (os_ - c * oz)) / (dz * os_ - ds * oz)
        z = oz + t * dz
        x, y = (None, other) if dim == 0 else (other, None)
        valid, m = _rule(x, y, z, t, np.abs(oz) + np.abs(t * dz))
    return t, valid, m


def _project(K, p, t):
    """project_camera_space of the camera-space points p, with validity and margin.  t is 0 or inf, always valid
    and exact: its test is no decision."""
    with np.errstate(invalid="ignore", divide="ignore"):
        q = _nan_to_num(p / (p[..., 2:] + EPS32), 1e8, -1e8)
    xy = q @ K[:2, :].T
    valid, m = _rule(xy[..., 0], xy[..., 1], p[..., 2], None, np.linalg.norm(p, axis=-1))
    assert t > -EPS_BOUNDS
    return valid, m


def overlap(extrinsics, intrinsics, h: int, w: int, src: int, dst: int) -> tuple[np.ndarray, np.ndarray, float]:
    """(overlaps [h*w] bool, margin [h*w], mask_margin) of the rays of frame `src` in the image of frame `dst`."""
    E = np.asarray(extrinsics, dtype=np.float64)
    K = np.asarray(intrinsics, dtype=np.float64)
    gx, gy = np.meshgrid((np.arange(w) + 0.5) / w, (np.arange(h) + 0.5) / h, indexing="xy")
    pix = np.stack([gx.reshape(-1), gy.reshape(-1), np.ones(h * w)], -1)
    dc = pix @ np.linalg.inv(K[src]).T
    dc = dc / np.linalg.norm(dc, axis=-1, keepdims=True)
    dw = dc @ E[src, :3, :3].T
    w2c = np.linalg.inv(E[dst])
    o = w2c[:3, :3] @ E[src, :3, 3] + w2c[:3, 3]
    d = dw @ w2c[:3, :3].T
    ob = np.broadcast_to(o, d.shape)
    Kd = K[dst]

    hits = [_frame_hit(Kd, ob, d, dim, val) for dim, val in ((0, 0.0), (0, 1.0), (1, 0.0), (1, 1.0))]
    ht, hv, hm = (np.stack([hh[i] for hh in hits]) for i in range(3))
    tlo, thi = np.where(hv, ht, np.inf), np.where(hv, ht, -np.inf)
    take = lambda a, i: np.take_along_axis(a, i[None], 0)[0]
    lo_v, hi_v = take(hv, np.argmin(tlo, 0)), take(hv, np.argmax(thi, 0))

    scale = max(1.0, float(np.linalg.norm(E[src, :3, 3])) + float(np.linalg.norm(E[dst, :3, 3])))
    norm_o = float(np.linalg.norm(o))
    at_camera = norm_o < EPS_BOUNDS
    zv, zm = _project(Kd, d if at_camera else ob, 0.0)
    if o[2] < EPS_BOUNDS and not at_camera:
        zv = np.zeros_like(zv)
    iv, im = _project(Kd, d, np.inf)
    overlaps = (zv | lo_v) & (iv | hi_v)

    TAU_SIDE = 1e-6        # an end projection this close to its rule may go either way: its side's hits count
    frame_m = hm.min(0)
    with np.errstate(invalid="ignore"):                 # inf - inf where fewer than two hits are valid: no tie
        srt = np.sort(tlo, 0)
        gap_lo = _rel(srt[1] - srt[0], srt[0])
        srt = np.sort(thi, 0)
        gap_hi = _rel(srt[-1] - srt[-2], srt[-1])
    lo_side = np.where(~zv | (zm < TAU_SIDE), np.minimum(frame_m, gap_lo), np.inf)
    hi_side = np.where(~iv | (im < TAU_SIDE), np.minimum(frame_m, gap_hi), np.inf)
    mask_margin = min(abs(o[2] - EPS_BOUNDS), abs(norm_o - EPS_BOUNDS)) / scale
    return overlaps, np.minimum.reduce([zm, im, lo_side, hi_side]), mask_margin


def pair_counts(extrinsics, intrinsics, h: int, w: int, context: int, k: int, tau: float):
    """((count_a, count_b), (flagged_a, flagged_b)): count_a is the rays of k in the image of `context`, count_b
    the rays of `context` in the image of k, as ps_view_overlap orders them; a ray is flagged when its margin is
    below tau or its pair's mask margin below MASK_TOL."""
    counts, flagged = [], []
    for src, dst in ((k, context), (context, k)):
        ov, m, mm = overlap(extrinsics, intrinsics, h, w, src, dst)
        counts.append(int(ov.sum()))
        flagged.append(h * w if mm < MASK_TOL else int((m < tau).sum()))
    return tuple(counts), tuple(flagged)
