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


# ---------------------------------------------------------------- settled pixels: parity with no anonymous allowance
# check_forward / check_backward forgive a fixed fraction of the data (0.1 % of pixels, the top 0.1 % of gradient
# entries) because a pixel whose alpha or transmittance sits on a decision threshold may go the other way on the
# GPU.  Nothing there checks that the forgiven data is that.  Here the oracle names the pixels that have a decision
# within SETTLED_DELTA of its threshold (oracle/raster_oracle.py decision_margins); every other pixel ("settled")
# is held element-wise, and the backward zeroes dL/dC on the unsettled pixels, so that they contribute exactly
# nothing on either side (every term of the composite backward, the background term included, is a multiple of
# its pixel's dL/dC) and EVERY gradient entry is held element-wise: no quantile anywhere.
SETTLED_DELTA = 1e-4      # relative margin on alpha / (1/255) and test_T / 1e-4 (ro.POWER_DELTA absolute on power)
SETTLED_COLOR_TOL, SETTLED_T_TOL = 2e-5, 1e-5
KINDS = ("alpha", "T", "power")


class SettledRef:
    """What the settled-pixel checks compare one view against: the float32 oracle forward (`f`), the float64
    composite on its records (`f64`), the decision margins, which pixels they leave unsettled and why."""

    def __init__(self, a, bg, H, W, delta=SETTLED_DELTA, fwd=None):
        self.a, self.bg, self.H, self.W, self.delta = a, bg, H, W, delta
        self.f = fwd if fwd is not None else oracle_forward(a, bg, W, H)
        self.f64 = ro.composite64_on_records(self.f, bg, W, H)
        self.margins = ro.decision_margins(self.f, W, H)
        self.kinds = ro.unsettled_kinds(self.margins, delta)
        self.settled = ro.settled_mask(self.margins, delta)
        self._grads = {}

    def counts(self) -> dict:
        return dict(pixels=self.settled.size, unsettled=int((~self.settled).sum()),
                    **{k: int(self.kinds[k].sum()) for k in KINDS})

    def d_img(self, seed=1):
        """Seeded dL/dC [3, H, W], zero on the unsettled pixels."""
        d = np.random.default_rng(seed).standard_normal((3, self.H, self.W)).astype(np.float32)
        return d * self.settled[None]

    def gradients(self, seed=1):
        """(float32 oracle, float64-composite-on-float32-records oracle) gradients for d_img(seed), cached."""
        if seed not in self._grads:
            a, d = self.a, self.d_img(seed)
            use_sh = a["sh"] is not None
            unpack = lambda b: dict(means=b.dL_dmeans, cov=b.dL_dcov6, opac=b.dL_dopacity,
                                    col=b.dL_dsh if use_sh else b.dL_dcolors, m2d=b.dL_dmean2D)
            n = lambda t: None if t is None else t.detach().cpu().numpy()
            b64 = ro.backward(self.f64, d, n(a["means"]), n(a["cov6"]), n(a["sh"]), n(a["vm"]), n(a["pm"]),
                              n(a["campos"]), a["tanfovx"], a["tanfovy"], np.asarray(self.bg, np.float64), self.W,
                              self.H, a["sh_degree"])
            self._grads[seed] = (unpack(oracle_backward(self.f, a, d, self.bg, self.W, self.H)), unpack(b64))
        return self._grads[seed]


def element_ratio(got: np.ndarray, ref: np.ndarray):
    """The mixed element bar of grad_errors at its MAXIMUM: (max over every entry of |got - ref| /
    (GRAD_ATOL_REL max|ref| + GRAD_RTOL |ref|), flat index of that entry)."""
    got, ref = np.asarray(got, np.float64).ravel(), np.asarray(ref, np.float64).ravel()
    if ref.size == 0:
        return 0.0, -1
    scale = max(float(np.abs(ref).max()), 1e-30)
    mixed = np.abs(got - ref) / (GRAD_ATOL_REL * scale + GRAD_RTOL * np.abs(ref))
    i = int(mixed.argmax())
    return float(mixed[i]), i


def describe_pixel(ref: SettledRef, y, x, got_n=None) -> str:
    """Where a pixel sits and how its walk went: what a failure message needs to find the kernel path."""
    f, gx = ref.f, (ref.W + 15) // 16
    tile = (y // 16) * gx + x // 16
    s, e = (int(v) for v in f.binned.ranges[tile])
    m = ref.margins
    return (f"pixel (y={y}, x={x}) tile {tile} (8x4 block row {(y % 16) // 4} col {(x % 16) // 8}, lane {(y % 4) * 8 + x % 8}) "
            f"list length {e - s}, n_contrib oracle {int(f.n_contrib[y, x])}"
            + ("" if got_n is None else f" native {int(got_n[y, x])}")
            + f", final_T {float(f.final_T[y, x]):.3e}, margins alpha {float(m.alpha[y, x]):.2e} "
            f"T {float(m.T[y, x]):.2e} power {float(m.power[y, x]):.2e}")


def compare_settled_forward(ref: SettledRef, color, n_contrib, final_T, tag="") -> dict:
    """One view's native colour [3,H,W], n_contrib and final_T [H,W] against the float32 oracle: on EVERY settled
    pixel n_contrib equal, |colour diff| <= SETTLED_COLOR_TOL, |final_T diff| <= SETTLED_T_TOL; on the unsettled
    ones <= 1e-2.  A pixel that is wrong and not unsettled fails with its coordinates and walk."""
    f, ok = ref.f, ref.settled
    diff = np.abs(color.astype(np.float64) - f.color).max(0)
    dT = np.abs(final_T.astype(np.float64) - f.final_T)
    n_ne = n_contrib.astype(np.int64) != f.n_contrib.astype(np.int64)
    wrong = n_ne | (diff > SETTLED_COLOR_TOL) | (dT > SETTLED_T_TOL)
    # the largest margin at which the GPU really decided differently: how much of SETTLED_DELTA it needs
    reach = np.minimum(ref.margins.alpha, ref.margins.T)[wrong & ~ref.kinds["power"]]
    rep = dict(ref.counts(), wrong_unsettled=int((wrong & ~ok).sum()), wrong_reach=float(reach.max()) if reach.size else 0.0,
               color=float(diff[ok].max()) if ok.any() else 0.0, final_T=float(dT[ok].max()) if ok.any() else 0.0,
               color_unsettled=float(diff[~ok].max()) if (~ok).any() else 0.0)
    print("SETTLED_FWD", tag, " ".join(f"{k}={v:.2e}" if isinstance(v, float) else f"{k}={v}" for k, v in rep.items()))
    bad = np.argwhere(wrong & ok)
    assert bad.size == 0, (f"{tag}: {len(bad)} settled pixels differ from the oracle (delta {ref.delta:g}); first: "
                           + "; ".join(describe_pixel(ref, int(y), int(x), n_contrib)
                                       + f" colour diff {diff[y, x]:.2e} T diff {dT[y, x]:.2e}" for y, x in bad[:4]))
    assert rep["color_unsettled"] <= 1e-2 and float(dT.max()) <= 1e-2, rep
    return rep


def check_forward_settled(ref: SettledRef, sort_impl=0, sh_basis=None, tag=""):
    """The CUDA forward of ref's view: check_forward (bit-exact front end, the loose image bars), then
    compare_settled_forward.  Returns (report, native colour)."""
    states = []
    _, color = check_forward(ref.a, ref.bg, ref.H, ref.W, sort_impl=sort_impl, sh_basis=sh_basis, fwd=ref.f,
                             states=states)
    im = states[0].intermediates()
    return compare_settled_forward(ref, color, im["n_contrib"][0].cpu().numpy(), im["final_T"][0].cpu().numpy(),
                                   tag), color


F64_BAR_FACTOR = 2.0     # vs the float64 reference: at most this times the float32 oracle's own worst ratio, or 1


def compare_settled_gradients(got: dict, ref32: dict, ref64: dict, tag="") -> dict:
    """Every entry of every tensor of `got` against the float32 oracle (element_ratio <= 1) and against the float64
    composite on float32 records (<= max(1, F64_BAR_FACTOR x the float32 oracle's own ratio)).  dL/dC was zero on
    the unsettled pixels on every side, so nothing is exempt."""
    rep = {}
    for k in got:
        r32, i32 = element_ratio(got[k], ref32[k])
        r64, i64 = element_ratio(got[k], ref64[k])
        own, _ = element_ratio(ref32[k], ref64[k])
        rep[k] = dict(f32=r32, f64=r64, own=own)
        row = lambda i: int(i // max(int(np.prod(np.shape(ref32[k])[1:])), 1))
        assert r32 <= 1.0, (f"{tag}: d{k} of Gaussian {row(i32)} is {r32:.2f}x its bar from the float32 oracle: got "
                            f"{np.ravel(got[k])[i32]:.6e} ref {np.ravel(ref32[k])[i32]:.6e}", rep)
        assert r64 <= max(1.0, F64_BAR_FACTOR * own), (
            f"{tag}: d{k} of Gaussian {row(i64)} is {r64:.2f}x its bar from the float64 reference (float32 oracle's own "
            f"{own:.2f}): got {np.ravel(got[k])[i64]:.6e} ref {np.ravel(ref64[k])[i64]:.6e}", rep)
    print("SETTLED_BWD", tag, " ".join(f"{k}:f32={r['f32']:.2f},f64={r['f64']:.2f},own={r['own']:.2f}"
                                       for k, r in rep.items()))
    return rep


def check_backward_settled(ref: SettledRef, seed=1, sh_basis=None, tag=""):
    """Gradients of the CUDA path for ref.d_img(seed) against both oracles, every entry (compare_settled_gradients)."""
    _, _, _, g = native(ref.a, ref.bg, ref.H, ref.W, 0, ref.d_img(seed), sh_basis=sh_basis)
    assert np.all(g["m2d"][:, 2] == 0)
    got = dict(means=g["means"], cov=g["cov"], opac=g["opac"], col=g["col"], m2d=g["m2d"][:, :2])
    return compare_settled_gradients(got, *ref.gradients(seed), tag=tag)
