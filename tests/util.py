"""Shared helpers of the parity tests: build rasterizer arguments from a synthetic scene, run the
CPU oracle, compare."""
from __future__ import annotations

import contextlib

import numpy as np
import torch

from oracle import raster_oracle as ro
from oracle import raster_torch as rt
from pixelsplat_b200 import synthetic


def view_args(scene: synthetic.Scene, view: int = 0, use_sh: bool = True, scale_invariant=True):
    """Rasterizer-level arguments of one view (fp32, CPU), via the oracle's restatement of
    render_cuda's host code."""
    return rt.prepare_view(scene.means, scene.covariances, scene.harmonics, scene.opacities,
                           scene.extrinsics[view], scene.intrinsics[view], scene.near[view],
                           scene.far[view], dtype=torch.float32, scale_invariant=scale_invariant,
                           use_sh=use_sh)


def oracle_forward(a: dict, bg, W, H):
    n = lambda t: None if t is None else t.detach().cpu().numpy()
    return ro.forward(n(a["means"]), n(a["cov6"]), n(a["opac"]), n(a["sh"]), n(a["colors"]),
                      n(a["vm"]), n(a["pm"]), n(a["campos"]), a["tanfovx"], a["tanfovy"],
                      np.asarray(bg, np.float32), W, H, a["sh_degree"], dtype=np.float32)


def oracle_forward64(a: dict, bg, W, H):
    """The same view in float64 (inputs are the float32 values, widened): the yardstick of the gradient bars."""
    n = lambda t: None if t is None else t.detach().cpu().numpy().astype(np.float64)
    return ro.forward(n(a["means"]), n(a["cov6"]), n(a["opac"]), n(a["sh"]), n(a["colors"]),
                      n(a["vm"]), n(a["pm"]), n(a["campos"]), a["tanfovx"], a["tanfovy"],
                      np.asarray(bg, np.float64), W, H, a["sh_degree"], dtype=np.float64)


def oracle_backward(fwd, a: dict, d_img, bg, W, H):
    n = lambda t: None if t is None else t.detach().cpu().numpy()
    return ro.backward(fwd, np.asarray(d_img, np.float32), n(a["means"]), n(a["cov6"]), n(a["sh"]),
                       n(a["vm"]), n(a["pm"]), n(a["campos"]), a["tanfovx"], a["tanfovy"],
                       np.asarray(bg, np.float32), W, H, a["sh_degree"])


def upstream_keys_from_native(keys_i64: np.ndarray, tile_start: np.ndarray, tile_count: np.ndarray):
    """Native per-tile keys (depth_bits << 32 | gaussian) -> upstream's (tile << 32 | depth_bits,
    gaussian) pairs, for ONE view whose segments start at tile_start[0]."""
    k = keys_i64.astype(np.uint64)
    depth = k >> np.uint64(32)
    gauss = (k & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    tile_of = np.repeat(np.arange(tile_count.size, dtype=np.uint64), tile_count.astype(np.int64))
    return (tile_of << np.uint64(32)) | depth, gauss


def psnr(a: np.ndarray, b: np.ndarray) -> float:
    """compute_psnr of the reference (src/evaluation/metrics.py:11-19) for one image."""
    a, b = np.clip(a, 0, 1), np.clip(b, 0, 1)
    mse = float(((a - b) ** 2).mean())
    return float("inf") if mse == 0 else -10.0 * np.log10(mse)


# Gradient bars against the FLOAT64 oracle (VERDICT r1 item 2a).  One global max per tensor lets an entry 100x
# smaller than the largest be 20 % wrong, so two more views of the same difference:
#   l2   = ||got - ref||_2 / ||ref||_2                                  (norm-wise relative error)
#   q999 = 99.9th percentile of |got - ref| / (ATOL_REL * max|ref| + RTOL * |ref|)   (element-wise, mixed)
# The percentile (not the max) because a pixel whose alpha sits on the 1/255 or T < 1e-4 decision boundary
# may legitimately take the other branch in float32 (ex2.approx on the GPU vs float64 exp in the oracle) and
# moves the handful of Gaussians that touch it.
GRAD_ATOL_REL, GRAD_RTOL = 1e-5, 1e-3


def grad_errors(got: np.ndarray, ref: np.ndarray) -> dict:
    got, ref = np.asarray(got, np.float64).ravel(), np.asarray(ref, np.float64).ravel()
    d = np.abs(got - ref)
    scale = max(float(np.abs(ref).max()), 1e-30)
    mixed = d / (GRAD_ATOL_REL * scale + GRAD_RTOL * np.abs(ref))
    return dict(max=float(d.max() / scale), l2=float(np.linalg.norm(d) / max(np.linalg.norm(ref), 1e-30)),
                q999=float(np.quantile(mixed, 0.999)) if mixed.size else 0.0)


def rel_err(got: np.ndarray, ref: np.ndarray) -> float:
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-30))


# ---------------------------------------------------------------- CUDA path vs the oracle (needs a GPU)
DEV = "cuda:0"
L2_BAR = 1e-4   # ||got - ref||_2 / ||ref||_2 per gradient tensor, float32 oracle


@contextlib.contextmanager
def composite_variant(impl: int = 2, segments: int = 0, hit_lists: int = 2):
    """Selects a compositor variant (ps_set_option "composite_impl", "composite_segments", "composite_hit_lists")
    for the block.  A forward and its backward must both run inside it: the options are process-wide and a
    backward reads the split and the hit lists of the options in force.  Restores the automatic defaults
    (2, 0, 2) on the way out, also when the block fails."""
    from pixelsplat_b200 import _lib
    try:
        _lib.set_option("composite_impl", impl)
        _lib.set_option("composite_segments", segments)
        _lib.set_option("composite_hit_lists", hit_lists)
        yield
    finally:
        _lib.set_option("composite_impl", 2)
        _lib.set_option("composite_segments", 0)
        _lib.set_option("composite_hit_lists", 2)


def native(a, bg, H, W, sort_impl=0, d_img=None, sh_basis=None):
    """One view through rasterize_gaussians: (colour [3,H,W], radii, RasterOutputState, gradients | None)."""
    from pixelsplat_b200.rasterizer import rasterize_gaussians
    t = lambda x: x.to(DEV)
    leaves = dict(means=t(a["means"])[None].clone().requires_grad_(True),
                  cov=t(a["cov6"])[None].clone().requires_grad_(True),
                  opac=t(a["opac"])[None].clone().requires_grad_(True))
    use_sh = a["sh"] is not None
    col = (a["sh"] if use_sh else a["colors"])
    leaves["col"] = t(col)[None].clone().requires_grad_(True)
    P = a["means"].shape[0]
    m2d = torch.zeros(1, P, 3, device=DEV, requires_grad=True)
    states = []
    color, radii = rasterize_gaussians(
        leaves["means"], leaves["cov"], leaves["opac"], leaves["col"],
        viewmatrix=t(a["vm"])[None], projmatrix=t(a["pm"])[None], campos=t(a["campos"])[None],
        tanfov=torch.tensor([[a["tanfovx"], a["tanfovy"]]], device=DEV),
        background=torch.tensor([bg], dtype=torch.float32, device=DEV), image_shape=(H, W),
        views_per_scene=1, sh_degree=a["sh_degree"], use_sh=use_sh, sort_impl=sort_impl,
        state_out=states, means2d=m2d, sh_basis=sh_basis)
    grads = None
    if d_img is not None:
        (color * torch.as_tensor(d_img, device=DEV)[None]).sum().backward()
        grads = {k: v.grad[0].cpu().numpy() for k, v in leaves.items()}
        grads["m2d"] = m2d.grad[0].cpu().numpy()
    return color[0].detach().cpu().numpy(), radii[0].cpu().numpy(), states[0], grads


def check_forward(a, bg, H, W, sort_impl=0, sh_basis=None, fwd=None, states=None):
    """The CUDA forward of one view against the float32 oracle (`fwd`, computed here when not given): bit-exact
    front end, fp32 tolerance on the composite.  Appends the native state to `states` if given.  Returns
    (oracle forward, native colour)."""
    f = fwd if fwd is not None else oracle_forward(a, bg, W, H)
    color, radii, st, _ = native(a, bg, H, W, sort_impl, sh_basis=sh_basis)
    if states is not None:
        states.append(st)
    im = {k: (v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in st.intermediates().items()}
    vis = f.pre.radii > 0
    # ---- bit-exact integer / index work
    assert np.array_equal(radii, f.pre.radii)
    assert np.array_equal(im["radii"][0], f.pre.radii)
    assert np.array_equal(im["rect"][0][vis].astype(np.int32), f.pre.rect[vis])
    assert np.array_equal(im["depth"][0][vis].view(np.uint32), f.pre.depth[vis].view(np.uint32))
    counts = (f.binned.ranges[:, 1] - f.binned.ranges[:, 0]).astype(np.int64)
    assert np.array_equal(im["tile_count"][0].astype(np.int64), counts)
    assert im["num_instances"] == f.binned.keys.size
    nz = counts > 0
    assert np.array_equal(im["tile_start"][0][nz].astype(np.int64), f.binned.ranges[nz, 0].astype(np.int64))
    k_up, v_up = upstream_keys_from_native(im["keys"], im["tile_start"][0], im["tile_count"][0])
    assert np.array_equal(k_up, f.binned.keys), "sorted (tile|depth) keys differ"
    assert np.array_equal(v_up, f.binned.values), "sorted Gaussian indices differ"
    # ---- preprocess floats: IEEE-exact (no FMA on either side)
    assert np.array_equal(im["xy"][0][vis], f.pre.xy[vis])
    assert np.array_equal(im["conic_opacity"][0][vis], f.pre.conic_opacity[vis])
    assert np.array_equal(im["rgb"][0][vis], f.pre.rgb[vis])
    cl = im["clamped"][0][vis]
    assert np.array_equal(np.stack([(cl >> c) & 1 for c in range(3)], -1), f.pre.clamped[vis])
    # ---- composite: fp32 tolerance
    diff = np.abs(color - f.color)
    assert diff.max() <= 1e-2, diff.max()
    assert (diff <= 2e-5).mean() >= 0.999, (diff <= 2e-5).mean()
    assert psnr(color, f.color) > 60.0
    assert (im["n_contrib"][0].astype(np.int64) == f.n_contrib.astype(np.int64)).mean() >= 0.999
    assert np.abs(im["final_T"][0] - f.final_T).max() <= 1e-2
    return f, color


def oracle_gradients(a, bg, H, W, d_img, fwd=None, with_f64=True):
    """The oracle's gradients for the upstream colour gradient d_img: (float32 oracle, float64 oracle | None), each a
    dict means / cov / opac / col / m2d."""
    use_sh = a["sh"] is not None
    unpack = lambda b: dict(means=b.dL_dmeans, cov=b.dL_dcov6, opac=b.dL_dopacity,
                            col=b.dL_dsh if use_sh else b.dL_dcolors, m2d=b.dL_dmean2D)
    f = fwd if fwd is not None else oracle_forward(a, bg, W, H)
    ref32 = unpack(oracle_backward(f, a, d_img, bg, W, H))
    ref64 = unpack(oracle_backward(oracle_forward64(a, bg, W, H), a, d_img, bg, W, H)) if with_f64 else None
    return ref32, ref64


def check_backward(a, bg, H, W, seed=1, tol=2e-3, sh_basis=None, with_f64=True, fwd=None, refs=None):
    """Gradients of the CUDA path against the oracle, three views of the same difference per tensor
    (grad_errors): max-norm, norm-wise (l2) and the 99.9th percentile of a mixed abs/rel element bar.
      * vs the FLOAT32 oracle (same decisions almost everywhere; differs by ex2.approx, FMA contraction in the
        composite and the order of the atomic sums):  max <= 2e-3, l2 <= 1e-4, q999 <= 1;
      * vs the FLOAT64 oracle: a float32 rasterizer takes a different branch than float64 at a few radius /
        1/255 / T < 1e-4 boundaries -- the float32 ORACLE itself sits at l2 ~ 1e-3 from float64 on re10k-like
        scenes -- so the bar is relative to that: our error <= 1.5x the float32 oracle's own error.
    `refs` = oracle_gradients(...) for the same seed, when the caller caches them.  Returns the per-tensor reports
    {"f32": ..., "f64": ... | None}."""
    d_img = np.random.default_rng(seed).standard_normal((3, H, W)).astype(np.float32)
    _, _, _, g = native(a, bg, H, W, 0, d_img, sh_basis=sh_basis)
    assert np.all(g["m2d"][:, 2] == 0)
    got = dict(means=g["means"], cov=g["cov"], opac=g["opac"], col=g["col"], m2d=g["m2d"][:, :2])
    ref32, ref64 = refs if refs is not None else oracle_gradients(a, bg, H, W, d_img, fwd, with_f64)
    rep32 = {k: grad_errors(got[k], ref32[k]) for k in got}
    fmt = lambda rep: {k: {m: f"{v:.1e}" for m, v in r.items()} for k, r in rep.items()}
    print("grad errors vs f32 oracle:", fmt(rep32))
    for k, r in rep32.items():
        assert r["max"] <= tol and r["l2"] <= L2_BAR and r["q999"] <= 1.0, (k, fmt(rep32))
    rep64 = None
    if with_f64:
        rep64 = {k: grad_errors(got[k], ref64[k]) for k in got}
        own = {k: grad_errors(ref32[k], ref64[k]) for k in got}
        print("grad errors vs f64 oracle:", fmt(rep64), "float32 oracle's own:", fmt(own))
        for k in got:
            assert rep64[k]["l2"] <= max(1.5 * own[k]["l2"], 1e-5), (k, fmt(rep64), fmt(own))
            assert rep64[k]["q999"] <= max(1.5 * own[k]["q999"], 1.0), (k, fmt(rep64), fmt(own))
    return {"f32": rep32, "f64": rep64}
