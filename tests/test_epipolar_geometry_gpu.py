"""The epipolar geometry kernel (csrc/epipolar_geometry.cu: k_epipolar_geometry behind ps_epipolar_geometry) against
the float64 restatement tests/epipolar_geometry_f64.py in "kernel" mode, fed the same float32 cameras widened to
float64, across its descriptor space.  The kernel is called through ctypes into buffers with a guard region after
each output.

The sweep is pairwise over grids 1x1, 1x7, 7x1, 6x10, 11x13, 16x16 (exactly two blocks of 128 rays), 33x65, 64x64;
S in {1, 2, 7, 32, 33, 64}; views 2, 3, 4, 5, 9, 33 (the other-view mapping ov < v ? ov : ov + 1 needs v >= 4);
batch 1-3; and the rigs of golden_util.camera_rig: generic, parallel, diverging, epipole, partial (valid and invalid
rays mixed in each view), facing (anti-parallel rays through the epipole), nearfar (near / far per (batch, view))
and aniso (fx != fy, principal point far from 0.5).

Elements within FLAG_TAU (relative) of a discrete decision of the restatement -- an in-bounds, in-front or
positive-t test of a projection that can become a segment end, a tie of frame-hit t, the parallel threshold -- or
with 1 + c < ANTIPARALLEL_TAU are excused; nothing else is.  On every case:
  valid          exact on every unflagged ray; flagged rays at most FLAGGED_RAYS_MAX of the call, flagged samples
                 at most FLAGGED_SAMPLES_MAX
  segments       exactly 0 on invalid rays; within 1 float32 ulp of the restatement rounded to float32 on valid ones
  rel_disparity  finite and in [0, 1] everywhere, flagged elements included; within 1 ulp on unflagged samples, and
                 bit-identical on at least BIT_IDENTICAL_MIN of them
  t_range        on valid unflagged rays |got - ref| <= T_RANGE_BAR * max(1, |ref|)
  coverage       every output element written (prefilled NaN / 0xAB), no guard element touched
Errors are reported per (batch, view, other view) slice, so a swapped camera shows even where a norm would hide it.
Two calls give the same bits, and a call replayed from a CUDA graph equals the eager call.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, over the 22 cases: no ray flagged; at most 12 of
3.1 M samples flagged (aniso 64x64), the largest share 7.6e-6 (2 of 262 144, generic 64x64); every unflagged segment
end and every unflagged rel_disparity bit-identical to the restatement rounded to float32 (0 ulp; the bars keep the
1 ulp allowance and 99.99 % bit identity for a different float64 evaluation order); t_range within 5.9e-8 relative
(its float32 rounding).  The file takes about 15 s.  With the sample position contracted into two FMAs, as this
kernel formed it before, 15 of the 22 cases fail: rel_disparity up to 2.7e3 ulp (2.3e-6) off on unflagged samples,
and bit-identical on as few as 92 % of them.
"""
import ctypes

import numpy as np
import pytest
import torch

from tests import epipolar_geometry_f64 as ref
from tests import golden_util as gu

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GUARD = 256

FLAG_TAU, ANTIPARALLEL_TAU = 1e-9, 1e-6
FLAGGED_RAYS_MAX, FLAGGED_SAMPLES_MAX = 1e-3, 3e-5
BIT_IDENTICAL_MIN = 0.9999
T_RANGE_BAR = 2e-7

# name -> (rig, b, v, (h, w), S)
CASES = {
    "generic-b1-v2-1x1-s1": ("generic", 1, 2, (1, 1), 1),
    "parallel-b2-v3-1x7-s2": ("parallel", 2, 3, (1, 7), 2),
    "diverging-b3-v2-7x1-s7": ("diverging", 3, 2, (7, 1), 7),
    "epipole-b1-v4-6x10-s32": ("epipole", 1, 4, (6, 10), 32),
    "partial-b2-v5-11x13-s33": ("partial", 2, 5, (11, 13), 33),
    "facing-b3-v3-16x16-s64": ("facing", 3, 3, (16, 16), 64),
    "nearfar-b1-v9-33x65-s7": ("nearfar", 1, 9, (33, 65), 7),
    "aniso-b2-v4-64x64-s32": ("aniso", 2, 4, (64, 64), 32),
    "generic-b1-v33-1x7-s32": ("generic", 1, 33, (1, 7), 32),
    "partial-b1-v33-7x1-s1": ("partial", 1, 33, (7, 1), 1),
    "epipole-b2-v9-16x16-s2": ("epipole", 2, 9, (16, 16), 2),
    "facing-b1-v2-64x64-s33": ("facing", 1, 2, (64, 64), 33),
    "nearfar-b3-v2-1x7-s64": ("nearfar", 3, 2, (1, 7), 64),
    "aniso-b3-v5-1x1-s33": ("aniso", 3, 5, (1, 1), 33),
    "diverging-b2-v9-11x13-s64": ("diverging", 2, 9, (11, 13), 64),
    "generic-b1-v2-64x64-s32": ("generic", 1, 2, (64, 64), 32),
    "parallel-b1-v4-33x65-s7": ("parallel", 1, 4, (33, 65), 7),
    "aniso-b1-v3-16x16-s1": ("aniso", 1, 3, (16, 16), 1),
    "facing-b2-v33-1x1-s7": ("facing", 2, 33, (1, 1), 7),
    "nearfar-b2-v3-11x13-s2": ("nearfar", 2, 3, (11, 13), 2),
    "epipole-b3-v5-7x1-s64": ("epipole", 3, 5, (7, 1), 64),
    "partial-b1-v4-6x10-s7": ("partial", 1, 4, (6, 10), 7),
}


def _inputs(rig, b, v):
    return [t.to(DEV, torch.float32).contiguous() for t in gu.camera_rig(b, v, rig)]


def _outputs(b, v, grid, S):
    """Guarded output buffers: NaN (floats) and 0xAB (valid), GUARD elements past each output."""
    n = b * v * (v - 1) * grid[0] * grid[1]
    f = lambda m: torch.full((m + GUARD,), float("nan"), dtype=torch.float32, device=DEV)
    return dict(segments=f(4 * n), valid=torch.full((n + GUARD,), 0xAB, dtype=torch.uint8, device=DEV),
                rel_disparity=f(S * n), t_range=f(2 * n), n=n)


def _call(cams, b, v, grid, S, out, stream=None):
    from pixelsplat_b200 import _lib
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    s = (stream or torch.cuda.current_stream()).cuda_stream
    rc = _lib.lib.ps_epipolar_geometry(b, v, grid[0], grid[1], S, *[p(t) for t in cams], p(out["segments"]),
                                       p(out["valid"]), p(out["rel_disparity"]), p(out["t_range"]), ctypes.c_void_p(s))
    _lib.check(rc, "ps_epipolar_geometry")


def _ulps(got, want32):
    """|got - want| in float32 ulps of want (both float32)."""
    with np.errstate(invalid="ignore"):
        return np.abs(got.astype(np.float64) - want32.astype(np.float64)) / np.spacing(np.abs(want32)).astype(np.float64)


@pytest.fixture(scope="module")
def report():
    rows = {}
    yield rows
    print("\nepipolar geometry sweep:")
    for name, r in rows.items():
        print(f"  {name}: " + ", ".join(f"{k} {v}" for k, v in r.items()))


@pytest.mark.parametrize("name", list(CASES))
def test_geometry_matches_f64(name, report):
    rig, b, v, grid, S = CASES[name]
    cams = _inputs(rig, b, v)
    out = _outputs(b, v, grid, S)
    _call(cams, b, v, grid, S, out)
    torch.cuda.synchronize()
    n, ov = out["n"], v - 1
    R = grid[0] * grid[1]
    host = {k: out[k].cpu().numpy() for k in ("segments", "valid", "rel_disparity", "t_range")}

    # coverage: every element written, no guard element touched
    assert np.isnan(host["segments"][4 * n:]).all() and np.isnan(host["rel_disparity"][S * n:]).all()
    assert np.isnan(host["t_range"][2 * n:]).all() and (host["valid"][n:] == 0xAB).all()
    seg = host["segments"][:4 * n].reshape(b, v, ov, R, 4)
    valid_raw = host["valid"][:n].reshape(b, v, ov, R)
    rd = host["rel_disparity"][:S * n].reshape(b, v, ov, R, S)
    tr = host["t_range"][:2 * n].reshape(b, v, ov, R, 2)
    assert np.isin(valid_raw, (0, 1)).all() and not np.isnan(seg).any() and not np.isnan(tr).any()
    valid = valid_raw.astype(bool)

    g = ref.geometry(*cams, grid, S, mode="kernel")
    ray_flag, smp_flag = ref.flags(g, FLAG_TAU, FLAG_TAU, ANTIPARALLEL_TAU, 0.0)
    ok = ~ray_flag
    r = report.setdefault(name, {})
    r["flagged rays"] = f"{int(ray_flag.sum())}/{ray_flag.size}"
    r["flagged samples"] = f"{int(smp_flag.sum())}/{smp_flag.size}"
    r["valid"] = f"{valid.mean():.2f}"

    # rel_disparity: finite and in [0, 1] everywhere, flagged elements included
    assert np.isfinite(rd).all() and (rd >= 0).all() and (rd <= 1).all(), (rd.min(), rd.max())
    # per-slice errors
    seg_ulp = np.where((valid & ok)[..., None], _ulps(seg, g["segments"].astype(np.float32)), 0.0)
    rd_ulp = np.where(~smp_flag, _ulps(rd, g["rel_disparity"].astype(np.float32)), 0.0)
    rd_abs = np.where(~smp_flag, np.abs(rd - g["rel_disparity"]), 0.0)
    t_ref = g["t_range"]
    with np.errstate(invalid="ignore"):
        t_err = np.where((valid & ok)[..., None], np.abs(tr - t_ref) / np.maximum(1.0, np.abs(t_ref)), 0.0)
    per_slice = {k: a.reshape(b, v, ov, -1).max(-1) for k, a in
                 (("seg_ulp", seg_ulp), ("rd_ulp", rd_ulp), ("rd_abs", rd_abs), ("t_err", t_err))}
    worst = {k: (float(a.max()), tuple(int(i) for i in np.unravel_index(int(a.argmax()), a.shape)))
             for k, a in per_slice.items()}
    bits = float((rd == g["rel_disparity"].astype(np.float32))[~smp_flag].mean()) if (~smp_flag).any() else 1.0
    r.update({k: f"{e:.3g} at (b, v, ov) {s}" for k, (e, s) in worst.items()})
    r["rd bit-identical"] = f"{bits:.5f}"
    r["valid mismatches"] = int((valid != g["valid"])[ok].sum())

    assert ray_flag.mean() <= FLAGGED_RAYS_MAX and smp_flag.mean() <= FLAGGED_SAMPLES_MAX, r
    assert np.array_equal(valid[ok], g["valid"][ok]), "valid differs on unflagged rays"
    assert (seg[~valid] == 0).all(), "invalid rays must have zero segments"
    assert worst["seg_ulp"][0] <= 1, worst["seg_ulp"]
    assert worst["rd_ulp"][0] <= 1, worst["rd_ulp"]
    assert bits >= BIT_IDENTICAL_MIN, bits
    assert worst["t_err"][0] <= T_RANGE_BAR, worst["t_err"]


@pytest.mark.parametrize("name", ["partial-b2-v5-11x13-s33", "facing-b1-v2-64x64-s33", "generic-b1-v33-1x7-s32"])
def test_repeats_and_graph_replay_are_bit_identical(name):
    rig, b, v, grid, S = CASES[name]
    cams = _inputs(rig, b, v)
    a, c = _outputs(b, v, grid, S), _outputs(b, v, grid, S)
    _call(cams, b, v, grid, S, a)
    _call(cams, b, v, grid, S, c)
    keys = ("segments", "valid", "rel_disparity", "t_range")
    torch.cuda.synchronize()
    for k in keys:
        assert torch.equal(a[k].view(torch.uint8) if k != "valid" else a[k],
                           c[k].view(torch.uint8) if k != "valid" else c[k]), k
    gr = _outputs(b, v, grid, S)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        _call(cams, b, v, grid, S, gr, stream=side)
    graph.replay()
    torch.cuda.synchronize()
    for k in keys:
        assert torch.equal(a[k].view(torch.uint8) if k != "valid" else a[k],
                           gr[k].view(torch.uint8) if k != "valid" else gr[k]), k
