"""Every compositor variant against the oracle.  Which path runs depends on the batch size, the instance capacity or
a process-wide option (include/pixelsplat_b200.h ps_set_option):
  * the warp-task compositor with K = 1, 2 or 4 list runs per task, with or without the forward's hit lists;
  * the legacy CTA-per-tile compositor (raster_composite.cu).
Each variant is forced here and runs the scenes below through the bars of tests/util.check_forward /
check_backward.  The scenes sit on the edges of the run split: saturation inside a run j >= 1 (including the
guard band 1e-4 <= T T_k < 1.01e-4, where a run is replayed although the pixel does not stop), runs with no
entries, long runs, partial tiles and several views per call.  The (T, C) state the forward stores in front of
each run (the state the K > 1 backward starts from) is compared with a float64 restatement of the sequential
loop."""
import math

import numpy as np
import pytest
import torch

from pixelsplat_b200 import synthetic
from tests import util

pytestmark = pytest.mark.gpu

DEV = util.DEV
# name -> (composite_impl, composite_segments, composite_hit_lists)
VARIANTS = {"legacy": (1, 1, 0),
            "k1": (2, 1, 1), "k1-nohl": (2, 1, 0),
            "k2": (2, 2, 1), "k2-nohl": (2, 2, 0),
            "k4": (2, 4, 1), "k4-nohl": (2, 4, 0)}
STOP_T, GUARD_T, ALPHA_MIN = 1e-4, 1.01e-4, 1.0 / 255.0
STATE_TOL = 1e-5          # run state (T, C): absolute, away from decision boundaries


def _segments(name):
    return VARIANTS[name][1] if VARIANTS[name][0] == 2 else 1


def _report(name, scene, **errs):
    print("VARIANT_ERR", name, scene, " ".join(f"{k}={v:.2e}" for k, v in errs.items()))


@pytest.fixture(scope="module")
def cache():
    """Oracle results, computed once per module and shared by the seven variants."""
    return {}


def _memo(cache, key, fn):
    if key not in cache:
        cache[key] = fn()
    return cache[key]


# ------------------------------------------------------------------ float64 restatement of the sequential loop
def sequential_run_states(f, H, W, K, tiles=None):
    """(T, Cr, Cg, Cb) of every pixel in front of list runs 1..K-1, walking each pixel's tile list in the sorted
    order (f.binned, which check_forward pins bit-exact to the native keys) in float64 with the oracle's xy, conic,
    opacity and rgb.  Run k starts at k * ceil(chunks / K) * 32 (whole 32-entry chunks; empty when the list is
    shorter).  A pixel that stopped keeps its state.  Returns (states [K-1, H, W, 4], near [H, W], checked [H, W]):
    `near` marks pixels that met a decision (alpha vs 1/255, T (1 - alpha) vs 1e-4, power vs 0) within float32
    reach before the last run start, `checked` the pixels of the walked tiles."""
    xy = f.pre.xy.astype(np.float64)
    co = f.pre.conic_opacity.astype(np.float64)
    rgb = f.pre.rgb.astype(np.float64)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    out = np.zeros((K - 1, H, W, 4))
    near = np.zeros((H, W), bool)
    checked = np.zeros((H, W), bool)
    for tile in (range(gx * gy) if tiles is None else tiles):
        tx, ty = tile % gx, tile // gx
        ys, xs = np.mgrid[ty * 16:min(ty * 16 + 16, H), tx * 16:min(tx * 16 + 16, W)]
        ys, xs = ys.ravel(), xs.ravel()
        px, py = xs.astype(np.float64), ys.astype(np.float64)
        s, e = (int(v) for v in f.binned.ranges[tile])
        count = e - s
        chunks = (count + 31) // 32
        per = (chunks + K - 1) // K
        begins = [min(count, k * per * 32) for k in range(1, K)]
        T = np.ones(px.size)
        C = np.zeros((px.size, 3))
        done = np.zeros(px.size, bool)
        close = np.zeros(px.size, bool)
        k = 0
        for i in range(begins[-1] + 1):
            while k < K - 1 and begins[k] == i:
                out[k, ys, xs, 0], out[k, ys, xs, 1:] = T, C
                k += 1
            if k == K - 1 or done.all():
                break
            g = f.binned.values[s + i]
            dx, dy = xy[g, 0] - px, xy[g, 1] - py
            power = -0.5 * (co[g, 0] * dx * dx + co[g, 2] * dy * dy) - co[g, 1] * dx * dy
            alpha = np.minimum(0.99, co[g, 3] * np.exp(power))
            contrib = ~done & (power <= 0) & (alpha >= ALPHA_MIN)
            test_T = T * (1 - alpha)
            close |= ~done & ((np.abs(alpha - ALPHA_MIN) <= 1e-5 * ALPHA_MIN) |
                              ((alpha >= ALPHA_MIN) & (np.abs(power) <= 1e-5)) |
                              (contrib & (np.abs(test_T - STOP_T) <= 2e-4 * STOP_T)))
            stop = contrib & (test_T < STOP_T)
            blend = contrib & ~stop
            C += np.where(blend, alpha * T, 0.0)[:, None] * rgb[g]
            T = np.where(blend, test_T, T)
            done |= stop
        while k < K - 1:
            out[k, ys, xs, 0], out[k, ys, xs, 1:] = T, C
            k += 1
        near[ys, xs] = close
        checked[ys, xs] = True
    return out, near, checked


def check_run_states(cache, key, f, run_state, H, W, K, tiles=None):
    """run_state [3, H, W, 4] of one view (what the forward stored) against the restatement, slots 0..K-2.  At most
    1 % of the pixels (or 4) may sit on a decision boundary; the 30k-entry tile has 3 of 256."""
    ref, near, checked = _memo(cache, ("states", key, K, tiles), lambda: sequential_run_states(f, H, W, K, tiles))
    got = np.asarray(run_state[:K - 1], np.float64)
    err = np.abs(got - ref).max(axis=(0, 3))                 # [H, W]
    ok = checked & ~near
    assert near.sum() <= max(4, 0.01 * checked.sum()), ("too many pixels on a decision boundary", int(near.sum()))
    bad = np.argwhere(ok & (err > STATE_TOL))
    assert bad.size == 0, ("run state differs", K, bad[:8].tolist(), float(err[ok].max()))
    # the split really happened: some pixel is still blending at a run start
    assert (ref[..., 0][:, checked] < 1.0).any() or not (f.binned.ranges[:, 1] > f.binned.ranges[:, 0]).any()
    return float(err[ok].max()) if ok.any() else 0.0, int(near[checked].sum())


# ------------------------------------------------------------------ one view through a forced variant
def _forward(name, a, bg, H, W, f):
    """check_forward under the current variant; also checks that the variant's hit-list setting took effect."""
    states = []
    _, color = util.check_forward(a, bg, H, W, fwd=f, states=states)
    st = states[0]
    from pixelsplat_b200 import _lib
    assert (_lib.layout(st.desc).block_hits == 0) == (VARIANTS[name][2] == 0)
    im = st.intermediates()
    diff = np.abs(color - f.color)
    return color, {k: im[k][0].cpu().numpy() for k in ("run_state", "n_contrib", "final_T")}, diff


def _backward(cache, key, a, bg, H, W, f, with_f64=True):
    d_img = np.random.default_rng(1).standard_normal((3, H, W)).astype(np.float32)
    refs = _memo(cache, ("grads", key, with_f64), lambda: util.oracle_gradients(a, bg, H, W, d_img, f, with_f64))
    return util.check_backward(a, bg, H, W, seed=1, with_f64=with_f64, refs=refs)


def _grad_summary(rep):
    out = {f"g32_{m}": max(r[m] for r in rep["f32"].values()) for m in ("max", "l2", "q999")}
    if rep["f64"] is not None:
        out["g64_l2"] = max(r["l2"] for r in rep["f64"].values())
    return out


def _run_scene(cache, name, key, a, bg, H, W, backward=True, with_f64=True, states=True):
    f = _memo(cache, ("fwd", key), lambda: util.oracle_forward(a, bg, W, H))
    with util.composite_variant(*VARIANTS[name]):
        color, im, diff = _forward(name, a, bg, H, W, f)
        errs = dict(img_max=float(diff.max()), img_frac_over_2e5=float((diff > 2e-5).mean()))
        K = _segments(name)
        if states and K > 1:
            errs["state"], errs["state_near"] = check_run_states(cache, key, f, im["run_state"], H, W, K)
        if backward:
            errs.update(_grad_summary(_backward(cache, key, a, bg, H, W, f, with_f64)))
    _report(name, key, **errs)
    return f, color, im


# ------------------------------------------------------------------ scenes
def _config0():
    sc = synthetic.scene_random_frustum(seed=3)
    return util.view_args(sc), (0.1, 0.2, 0.3), *sc.image_shape


def _ragged():
    sc = synthetic.scene_random_frustum(seed=6, image_hw=(50, 70), num_gaussians=4000, z_range=(1.0, 4.0))
    return util.view_args(sc), (0.0, 0.0, 0.0), 50, 70


@pytest.mark.parametrize("name", list(VARIANTS))
def test_config0(cache, name):
    """configs[0]: 64x64, 1k Gaussians, non-zero background; forward, backward (float64 bar), run states."""
    _run_scene(cache, name, "config0", *_config0())


@pytest.mark.parametrize("name", list(VARIANTS))
def test_ragged_saturating(cache, name):
    """70x50 (partial tiles: lanes outside the image), 4k opaque Gaussians: early termination everywhere."""
    f, _, _ = _run_scene(cache, name, "ragged", *_ragged())
    assert (f.final_T < 1e-3).mean() > 0.05


# ---- saturation sweep: 256 copies of one Gaussian on one 16x16 tile, a colour ramp over the list index
SWEEP_L, SWEEP_HW = 256, 16
SWEEP_S2 = 56.25 / math.log(10.0)      # screen variance: alpha falls 10x from the centre to the corner pixel


def _sweep_args(opacity):
    """L Gaussians with the same mean (the image centre), covariance and depth; only the colour differs.  Every
    entry has the same alpha at a pixel: alpha(p) = opacity exp(-|p - c|^2 / (2 s^2)), s^2 = SWEEP_S2."""
    from oracle import raster_torch as rt
    W = H = SWEEP_HW
    Kmat = torch.tensor([[0.88, 0, 0.5], [0, 0.88, 0.5], [0, 0, 1.0]])
    vm, pm, cp, tx, ty = rt.camera_from_c2w(torch.eye(4), Kmat, 0.5, 100.0, torch.float32)
    z, focal = 5.0, W / (2 * tx)
    sigma = math.sqrt(SWEEP_S2 - 0.3) * z / focal          # the rasterizer adds 0.3 px^2 of low-pass filter
    i = torch.arange(SWEEP_L, dtype=torch.float32)
    colors = torch.stack([i / (SWEEP_L - 1), 1 - i / (SWEEP_L - 1), (i % 64) / 63], -1)
    return dict(means=torch.tensor([[0.0, 0.0, z]]).repeat(SWEEP_L, 1),
                cov6=torch.tensor([[sigma ** 2, 0, 0, sigma ** 2, 0, sigma ** 2]]).repeat(SWEEP_L, 1),
                opac=torch.full((SWEEP_L,), float(opacity)), sh=None, colors=colors.contiguous(),
                vm=vm, pm=pm, campos=cp, tanfovx=tx, tanfovy=ty, sh_degree=0)


def _sweep_alpha(f):
    """Per-pixel alpha (float64) of the sweep's Gaussian, from the oracle's screen position and conic."""
    ys, xs = np.mgrid[0:SWEEP_HW, 0:SWEEP_HW].astype(np.float64)
    (x, y), (ca, cb, cc, o) = f.pre.xy[0].astype(np.float64), f.pre.conic_opacity[0].astype(np.float64)
    dx, dy = x - xs, y - ys
    return np.minimum(0.99, o * np.exp(-0.5 * (ca * dx * dx + cc * dy * dy) - cb * dx * dy))


def _band_opacity(n):
    """Opacity that puts pixel (7, 7) at (1 - alpha)^n = 1.005e-4, the middle of the guard band."""
    f = util.oracle_forward(_sweep_args(0.5), (0, 0, 0), SWEEP_HW, SWEEP_HW)
    alpha = 1 - (1.005e-4) ** (1 / n)
    return alpha * 0.5 / _sweep_alpha(f)[7, 7]


def sweep_closed_form(alpha, colors, bg):
    """The sequential recurrence with equal alphas, in float64: entries 0 .. n-1 blend, where n is the first index
    with (1 - alpha)^(n+1) < 1e-4 (or L; 0 where alpha < 1/255).  Returns (image [3,H,W], final T, n_contrib, stop
    index or -1)."""
    L = colors.shape[0]
    n = np.arange(L + 1)
    skip = alpha < ALPHA_MIN
    alpha = np.where(skip, 0.0, alpha)
    Tn = (1 - alpha[..., None]) ** n                              # [H, W, L+1]: T in front of entry n
    stops = Tn[..., 1:] < STOP_T
    stop_at = np.where(stops.any(-1), stops.argmax(-1), -1)
    n_blend = np.where(skip, 0, np.where(stop_at >= 0, stop_at, L))
    w = np.where(n[None, None, :L] < n_blend[..., None], alpha[..., None] * Tn[..., :L], 0.0)
    C = np.einsum("hwl,lc->chw", w, colors.astype(np.float64))
    T = np.take_along_axis(Tn, n_blend[..., None], -1)[..., 0]
    return C + T[None] * np.asarray(bg, np.float64)[:, None, None], T, n_blend, stop_at


def _sweep_cases():
    return {"sweep": 0.3, "band128": _band_opacity(128), "band256": _band_opacity(256)}


def test_saturation_sweep_covers_every_run_and_the_guard_band(cache):
    """From the closed form alone: the sweep stops pixels inside runs 0, 1 and 2 of K = 4 and in both runs of K = 2,
    leaves some pixels unstopped, and the band scenes put a pixel's T T_k inside [1e-4, 1.01e-4) at a fold of
    K = 2 and of K = 4 (replayed without stopping)."""
    cases = _memo(cache, "sweep_cases", _sweep_cases)
    band = {2: False, 4: False}
    for key, o in cases.items():
        a = _sweep_args(o)
        f = _memo(cache, ("fwd", key), lambda: util.oracle_forward(a, (0, 0, 0), SWEEP_HW, SWEEP_HW))
        alpha = _sweep_alpha(f)
        _, _, _, stop_at = sweep_closed_form(alpha, a["colors"].numpy(), (0, 0, 0))
        if key == "sweep":
            assert 0.25 < alpha.max() < 0.35 and 0.02 < alpha.min() < 0.04
            assert set(np.unique(stop_at[stop_at >= 0] // 64)) >= {0, 1, 2}          # K = 4 runs
            assert set(np.unique(stop_at[stop_at >= 0] // 128)) == {0, 1}             # K = 2 runs
            assert (stop_at < 0).any()
        for K in (2, 4):
            for j in range(1, K):
                total = (1 - alpha) ** ((j + 1) * SWEEP_L // K)   # T in front of run j times run j's own T
                not_stopped = (1 - alpha) ** (j * SWEEP_L // K) >= STOP_T
                band[K] |= bool(((total >= STOP_T) & (total < GUARD_T) & not_stopped).any())
    assert band[2] and band[4], band


@pytest.mark.parametrize("name", list(VARIANTS))
def test_saturation_sweep(cache, name):
    """Known answer: the sweep scenes against the oracle and against the float64 closed form (image and T within
    5e-5 absolute -- ex2.approx moves alpha by ~1e-6 relative, compounded over up to 256 entries -- and n_contrib
    exact), forward, backward and run states."""
    cases = _memo(cache, "sweep_cases", _sweep_cases)
    bg = (0.05, 0.1, 0.15)
    for key, o in cases.items():
        a = _sweep_args(o)
        f, color, im = _run_scene(cache, name, key + "_bg", a, bg, SWEEP_HW, SWEEP_HW)
        img, T, n_blend, _ = sweep_closed_form(_sweep_alpha(f), a["colors"].numpy(), bg)
        e_img, e_T = float(np.abs(color - img).max()), float(np.abs(im["final_T"] - T).max())
        _report(name, key + "_closed_form", img=e_img, T=e_T)
        assert e_img <= 5e-5 and e_T <= 5e-5, (key, e_img, e_T)
        assert np.array_equal(im["n_contrib"].astype(np.int64), n_blend), key


@pytest.mark.parametrize("name", list(VARIANTS))
def test_short_lists_empty_and_single(cache, name):
    """40 Gaussians at 64x64: most tiles hold fewer than 32 K entries, so runs 1.. are empty.  Also nothing visible
    (all behind the camera) and a single Gaussian."""
    sc = synthetic.scene_random_frustum(seed=14, num_gaussians=40)
    f, _, _ = _run_scene(cache, name, "short", util.view_args(sc), (0.0, 0.0, 0.0), *sc.image_shape)
    cnt = f.binned.ranges[:, 1] - f.binned.ranges[:, 0]
    assert cnt.max() < 32 * 2 and (cnt > 0).sum() >= 4
    sc1 = synthetic.scene_random_frustum(seed=10, num_gaussians=1)
    sc1.means[0] = torch.tensor([0.0, 0.0, 3.0])
    _run_scene(cache, name, "single", util.view_args(sc1), (0.0, 0.0, 0.0), *sc1.image_shape)
    sc0 = synthetic.scene_random_frustum(seed=9, num_gaussians=64)
    sc0.means[:, 2] = -sc0.means[:, 2]
    a0, bg0 = util.view_args(sc0), (0.3, 0.4, 0.5)
    with util.composite_variant(*VARIANTS[name]):
        f0, color0 = util.check_forward(a0, bg0, 64, 64, fwd=_memo(cache, ("fwd", "culled"),
                                                                   lambda: util.oracle_forward(a0, bg0, 64, 64)))
        _, _, _, g = util.native(a0, bg0, 64, 64, 0, np.ones((3, 64, 64), np.float32))
    assert f0.binned.keys.size == 0
    assert np.allclose(color0, np.array(bg0, np.float32)[:, None, None])
    assert all(np.all(v == 0) for v in g.values())


@pytest.mark.parametrize("name", list(VARIANTS))
def test_long_lists(cache, name):
    """One 16x16 tile under 30k Gaussians: runs many chunks long.  Forward for every variant, backward (float32
    oracle) for K = 1 and K = 4."""
    sc = synthetic.scene_random_frustum(seed=7, image_hw=(16, 16), num_gaussians=30000, z_range=(2.0, 30.0))
    f, _, _ = _run_scene(cache, name, "long", util.view_args(sc), (0.0, 0.0, 0.0), 16, 16,
                         backward=_segments(name) in (1, 4) and name != "legacy", with_f64=False)
    assert f.binned.keys.size > 12288


# ---- several views per call
def _batched(scs, V, H, W, d_img):
    """S scenes x V views in one rasterize_gaussians call (shared Gaussians per scene, host-side cameras of
    util.view_args without the per-view rescale, so the oracle sees the same arguments).  Returns (colour
    [S, V, 3, H, W], state, per-scene gradients)."""
    from pixelsplat_b200.rasterizer import rasterize_gaussians
    S = len(scs)
    args = [[util.view_args(sc, view=v, scale_invariant=False) for v in range(V)] for sc in scs]
    st = lambda k: torch.stack([args[s][0][k] for s in range(S)]).to(DEV).requires_grad_(True)
    leaves = dict(means=st("means"), cov=st("cov6"), opac=st("opac"), col=st("sh"))
    cam = lambda k: torch.stack([args[s][v][k] for s in range(S) for v in range(V)]).to(DEV)
    states = []
    color, _ = rasterize_gaussians(
        leaves["means"], leaves["cov"], leaves["opac"], leaves["col"], viewmatrix=cam("vm"), projmatrix=cam("pm"),
        campos=cam("campos"),
        tanfov=torch.tensor([[args[s][v]["tanfovx"], args[s][v]["tanfovy"]] for s in range(S) for v in range(V)],
                            device=DEV),
        background=torch.zeros(S * V, 3, device=DEV), image_shape=(H, W), views_per_scene=V,
        sh_degree=args[0][0]["sh_degree"], state_out=states)
    (color * torch.as_tensor(d_img.reshape(S * V, 3, H, W), device=DEV)).sum().backward()
    grads = [{k: l.grad[s].cpu().numpy() for k, l in leaves.items()} for s in range(S)]
    return color.detach().cpu().numpy().reshape(S, V, 3, H, W), states[0], grads, args


def _batched_oracle(args, d_img, H, W):
    """Per view: the float32 oracle forward and its gradients; per scene: the gradients summed over views."""
    from concurrent.futures import ThreadPoolExecutor

    def job(sv):
        s, v = sv
        a = args[s][v]
        f = util.oracle_forward(a, (0, 0, 0), W, H)
        b = util.oracle_backward(f, a, d_img[s, v], (0, 0, 0), W, H)
        return f, dict(means=b.dL_dmeans, cov=b.dL_dcov6, opac=b.dL_dopacity, col=b.dL_dsh)

    S, V = len(args), len(args[0])
    with ThreadPoolExecutor(8) as ex:          # the C oracle releases the GIL
        res = list(ex.map(job, [(s, v) for s in range(S) for v in range(V)]))
    fwd = [[res[s * V + v][0] for v in range(V)] for s in range(S)]
    sums = [{k: sum(res[s * V + v][1][k] for v in range(V)) for k in res[0][1]} for s in range(S)]
    return fwd, sums


def _check_batched(cache, name, key, scs, V, H, W, sample_tiles):
    S = len(scs)
    d_img = np.random.default_rng(5).standard_normal((S, V, 3, H, W)).astype(np.float32)
    from pixelsplat_b200 import _lib
    with util.composite_variant(*VARIANTS[name]) if name else util.composite_variant():
        got, st, grads, args = _batched(scs, V, H, W, d_img)
        hl_on = _lib.layout(st.desc).block_hits != 0
        im = st.intermediates()
    fwd, sums = _memo(cache, ("batched", key), lambda: _batched_oracle(args, d_img, H, W))
    errs = dict(img_max=0.0, img_frac_over_2e5=0.0)
    n_contrib = im["n_contrib"].cpu().numpy()
    run_state = im["run_state"].cpu().numpy()
    K = _segments(name) if name else 2
    for s in range(S):
        for v in range(V):
            f = fwd[s][v]
            diff = np.abs(got[s, v] - f.color)
            assert diff.max() <= 1e-2 and (diff <= 2e-5).mean() >= 0.999, (s, v, diff.max())
            assert util.psnr(got[s, v], f.color) > 60.0
            assert (n_contrib[s * V + v].astype(np.int64) == f.n_contrib.astype(np.int64)).mean() >= 0.999
            errs["img_max"] = max(errs["img_max"], float(diff.max()))
            errs["img_frac_over_2e5"] = max(errs["img_frac_over_2e5"], float((diff > 2e-5).mean()))
            if K > 1:   # per-view run-state indexing: (vid * 3 + run - 1) * H * W
                e, _ = check_run_states(cache, (key, s, v), f, run_state[s * V + v], H, W, K, tiles=sample_tiles)
                errs["state"] = max(errs.get("state", 0.0), e)
    for s in range(S):
        for k in ("means", "cov", "opac", "col"):
            r = util.grad_errors(grads[s][k], sums[s][k])
            assert r["max"] <= 2e-3 and r["l2"] <= util.L2_BAR and r["q999"] <= 1.0, (s, k, r)
            for m in ("max", "l2", "q999"):
                errs[f"g32_{m}"] = max(errs.get(f"g32_{m}", 0.0), r[m])
    _report(name or "auto", key, **errs)
    return hl_on


@pytest.mark.parametrize("name", list(VARIANTS))
def test_batched_views(cache, name):
    """S = 2 scenes x V = 2 views at 128x128 in one call (unforced this selects K = 4): every view against the
    oracle, the view-summed gradients of both scenes, and the run states of sampled tiles of every view."""
    scs = [synthetic.scene_re10k_like(seed=80 + i, image_hw=(128, 128), target_views=2) for i in range(2)]
    _check_batched(cache, name, "s2v2_128", scs, 2, 128, 128, sample_tiles=(0, 9, 27, 36, 54, 63))


def test_automatic_two_runs():
    """The production K = 2 shape, nothing forced: one scene, two 256x256 views per call (exactly 4096 warp tasks).
    The run states of sampled tiles match the K = 2 split (not K = 4's), and the hit lists are kept."""
    scs = [synthetic.scene_re10k_like(seed=90, image_hw=(256, 256), target_views=2)]
    assert _check_batched({}, None, "s1v2_256", scs, 2, 256, 256, sample_tiles=(0, 77, 136, 255))


@pytest.mark.parametrize("name", ["k1", "k2", "k2-nohl"])
def test_config1_forced_runs(cache, name):
    """configs[1] (256x256, P = 393 216) with K = 1 and K = 2 forced: forward and backward against the float32
    oracle."""
    sc = synthetic.scene_re10k_like(seed=0)
    _run_scene(cache, name, "config1", util.view_args(sc), (0.0, 0.0, 0.0), 256, 256, with_f64=False, states=False)


def test_options_are_back_at_their_defaults():
    """After the module: a 256x256 desc whose capacity is below the 512 MB threshold keeps its hit lists."""
    from pixelsplat_b200 import _lib
    d = _lib.RasterDesc(1, 1, 393216, 25, 4, 0, 0, 256, 256, 0, 0, 3 * 393216)
    assert _lib.layout(d).block_hits != 0
