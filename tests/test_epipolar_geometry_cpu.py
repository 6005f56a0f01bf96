"""The float64 restatement of the epipolar geometry (tests/epipolar_geometry_f64.py) against the reference's own
float64 outputs (tests/golden/epipolar_geometry.npz and epipolar_geometry_v2.npz, oracle/make_epipolar_golden.py),
on every golden case: the restatement is the yardstick of tests/test_epipolar_geometry_gpu.py, so it must be the
reference's math.

  reference mode  valid exact; segments, t_min / t_max and rel_disparity within REF_BAR (the reference solves the
                  closest point by lstsq, the restatement in closed form: measured worst 1.0e-12 on rel_disparity
                  (epipole), 5.7e-15 on the segments); only elements within FLAG_TAU of a decision are excused: no
                  ray and one sample (model64) on these cases
  kernel mode     (float32 cameras, float32 sample positions) within the bars the GPU kernel was held to against the
                  same goldens before the restatement existed (tests/test_epipolar_gpu.py)
"""
from pathlib import Path

import numpy as np
import pytest
import torch

from tests import epipolar_geometry_f64 as ref
from tests import golden_util as gu

GOLD = Path(__file__).resolve().parent / "golden"
REF_BAR = 4e-12
FLAG_TAU = 1e-9

# name -> (rig, b, v, grid, S, file, key prefix)
CASES = {
    "generic": ("generic", 2, 2, (8, 8), 32, "epipolar_geometry.npz", "generic_f64_"),
    "parallel": ("parallel", 1, 3, (8, 8), 32, "epipolar_geometry.npz", "parallel_f64_"),
    "diverging": ("diverging", 1, 2, (8, 8), 32, "epipolar_geometry.npz", "diverging_f64_"),
    "generic3": ("generic", 1, 3, (6, 10), 32, "epipolar_geometry.npz", "generic3_f64_"),
    "model64": ("generic", 1, 2, (64, 64), 32, "epipolar_geometry_v2.npz", "model64_"),
    "b2v3": ("generic", 2, 3, (11, 13), 32, "epipolar_geometry_v2.npz", "b2v3_"),
    "epipole": ("epipole", 2, 3, (8, 8), 32, "epipolar_geometry_v2.npz", "epipole_"),
    "partial": ("partial", 2, 3, (8, 8), 32, "epipolar_geometry_v2.npz", "partial_"),
    "facing": ("facing", 2, 3, (8, 8), 32, "epipolar_geometry_v2.npz", "facing_"),
    "nearfar": ("nearfar", 2, 3, (8, 8), 32, "epipolar_geometry_v2.npz", "nearfar_"),
}


def _gold(name):
    rig, b, v, grid, S, fname, pre = CASES[name]
    g = np.load(GOLD / fname)
    out = {k[len(pre):]: g[k] for k in g.files if k.startswith(pre)}
    out["stride"] = int(out.get("stride", 1))
    return out


def _flags(g):
    return ref.flags(g, FLAG_TAU, FLAG_TAU, FLAG_TAU, 0.0)


@pytest.mark.parametrize("name", list(CASES))
def test_reference_mode_matches_reference(name):
    rig, b, v, grid, S, _, _ = CASES[name]
    gold = _gold(name)
    g = ref.geometry(*gu.camera_rig(b, v, rig), grid, S, mode="reference")
    ray_flag, smp_flag = _flags(g)
    st = gold["stride"]
    print(name, "flagged rays", int(ray_flag.sum()), "of", ray_flag.size, "samples", int(smp_flag.sum()))
    assert ray_flag.mean() < 0.01
    ok = ~ray_flag
    assert np.array_equal(g["valid"][ok], gold["valid"].astype(bool)[ok])
    e_seg = np.abs(g["segments"] - gold["segments"])[ok].max()
    e_rd = np.abs(g["rel_disparity"][..., ::st, :] - gold["rel_disparity"])[~smp_flag[..., ::st, :]].max()
    print(name, "segments", e_seg, "rel_disparity", e_rd)
    assert e_seg < REF_BAR and e_rd < REF_BAR
    if "t_min" in gold:
        vr = g["valid"] & ok
        for i, k in enumerate(("t_min", "t_max")):
            e = np.abs(g["t_range"][..., i][vr] - gold[k][vr]) / np.maximum(1.0, np.abs(gold[k][vr]))
            assert e.max(initial=0.0) < REF_BAR, (k, e.max())


@pytest.mark.parametrize("name", ["generic", "parallel", "diverging", "generic3"])
def test_kernel_mode_meets_the_gpu_bars(name):
    """On float32 cameras, widened, with float32 sample positions: the restatement of what the kernel computes meets
    the bars the kernel meets against the float64 reference on the cases those bars were set on.  (On the new cases
    the float32 rounding of the cameras moves near-parallel depths further: up to 8e-4 on model64.)"""
    rig, b, v, grid, S, _, _ = CASES[name]
    gold = _gold(name)
    cams = [t.to(torch.float32) for t in gu.camera_rig(b, v, rig)]
    g = ref.geometry(*cams, grid, S, mode="kernel")
    assert np.array_equal(g["valid"], gold["valid"].astype(bool))
    assert np.abs(g["segments"] - gold["segments"]).max() < 2e-6
    err = np.abs(g["rel_disparity"][..., ::gold["stride"], :] - gold["rel_disparity"])
    assert np.quantile(err, 0.99) < 5e-6 and err.max() < 5e-4, (np.quantile(err, 0.99), err.max())


def test_kernel_mode_rounds_the_sample_like_float32():
    """Kernel mode forms xy_s = f32(x0 + f32(u * f32(x1 - x0))) from the float32 segment ends: every sample is a
    float32 value, and on the golden segments a fused multiply-add (one rounding) differs from it by an ulp on a few
    per cent of the coordinates, which is what this mode must not do."""
    g = ref.geometry(*[t.to(torch.float32) for t in gu.camera_rig(2, 2, "generic")], (8, 8), 32, mode="kernel")
    xy = g["xy_sample"]
    assert np.array_equal(xy.astype(np.float32).astype(np.float64), xy)
    seg = g["segments"].astype(np.float32).astype(np.float64)
    u = ((np.arange(32) + 0.5) / 32).astype(np.float32).astype(np.float64)
    fused = (seg[..., None, :2] + u[:, None] * (seg[..., None, 2:] - seg[..., None, :2]).astype(np.float32))
    fused = fused.astype(np.float32).astype(np.float64)
    frac = float((fused != xy)[g["valid"]].mean())
    print("fused-vs-rounded sample differs on", frac)
    assert 0.0 < frac < 0.2


def test_rigs():
    """The rigs do what camera_rig says they do."""
    for rig in ("partial",):
        for v in (2, 3):
            g = ref.geometry(*gu.camera_rig(2, v, rig), (8, 8), 4, mode="reference")
            frac = g["valid"].mean(-1)
            assert ((frac > 0.05) & (frac < 0.95)).all(), frac       # every slice mixes valid and invalid rays
    g = ref.geometry(*gu.camera_rig(1, 2, "facing"), (64, 64), 32, mode="reference")
    assert g["sample_margins"]["antiparallel"].min() < 1e-3          # rays through the epipole: near anti-parallel
    _, _, near, far = gu.camera_rig(2, 3, "nearfar")
    assert len(set(near.reshape(-1).tolist())) == 6 and len(set(far.reshape(-1).tolist())) == 6
    _, K, _, _ = gu.camera_rig(2, 3, "aniso")
    assert (K[..., 0, 0] / K[..., 1, 1] > 1.5).all() and (abs(K[..., :2, 2] - 0.5) > 0.25).all()
