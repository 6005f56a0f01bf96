"""CPU tests of the settled-pixel instrument (oracle/raster_oracle.py decision_margins, settled_mask,
composite64_on_records; tests/util.py SettledRef and the compare_settled_* helpers), before it is pointed at the GPU.

  * hand-built cases: a Gaussian whose alpha at one pixel is (1/255)(1 +- eps), a stack whose T (1 - alpha) at one
    pixel is 1e-4 (1 +- eps), eps either side of delta; a conic whose power cancels to 0 or just above;
  * on the scenes of tests/test_settled_pixels_gpu.py: the float32 oracle and the float64 composite on the float32
    records take the same decisions on EVERY settled pixel (the evidence that delta is above float32 rounding of the
    decision values) and, with dL/dC zero on the unsettled pixels, agree on every gradient entry.  Measured: the mixed
    element ratio |d| / (1e-5 max|ref| + 1e-3 |ref|) of the float32 oracle against the float64 reference reaches at
    most 0.023 (covariance gradient, the 256x256 RE10k-like scene); the bar here is 0.05;
  * the comparison's own sensitivity: a planted error on 0.05 % of the settled pixels and in the gradient rows of
    0.05 % of the Gaussians (3 x their bar) passes the percentile bars of check_forward / grad_errors and fails the settled ones.

Unsettled fractions (printed by the scene test for delta = 1e-5, 1e-4, 1e-3): at delta = 1e-4 between 0 and 0.8 % of
a view's pixels (0.75 % on the 256x256 RE10k-like scene, nearly all alpha-vs-1/255; 2.1 % on the 512x512 scene, which only the GPU test runs); at 1e-3 it would be 3 - 7 %."""
import numpy as np
import pytest

from oracle import raster_oracle as ro
from tests import test_oracle_raster as tor
from tests import util
from tests.test_settled_pixels_gpu import MAX_UNSETTLED, SCENES

DELTA = util.SETTLED_DELTA
CPU_SCENES = [k for k in SCENES if k != "config4"]      # 512x512: minutes of float64 oracle; the GPU test covers it
OWN_BAR = 0.05
_REFS = {}


def _ref(key) -> util.SettledRef:
    if key not in _REFS:
        _REFS[key] = util.SettledRef(*SCENES[key]())
    return _REFS[key]


def _falloff(f, g, x, y):
    """exp(power) of Gaussian g at pixel (x, y), float64, from the oracle's records."""
    (cx, cy), (a, b, c, _) = f.pre.xy[g].astype(np.float64), f.pre.conic_opacity[g].astype(np.float64)
    dx, dy = cx - x, cy - y
    return float(np.exp(-0.5 * (a * dx * dx + c * dy * dy) - b * dx * dy))


@pytest.mark.parametrize("sign", [+1, -1])
@pytest.mark.parametrize("eps", [0.5 * DELTA, 2 * DELTA])
def test_alpha_margin_of_one_gaussian(sign, eps):
    """One Gaussian centred off the pixel grid (no two pixels share a distance), opacity tuned so that alpha at pixel
    (24, 31) is (1/255)(1 + sign eps): that pixel's alpha margin is eps, it blends iff sign > 0, it is unsettled iff
    eps <= delta, and every other pixel is settled."""
    W = H = 64
    x, y = 24, 31
    _, _, _, tx, ty = tor._identity_camera(W, H)
    p = tor._point_for_pixel(20.3, 30.2, 5.0, W, H, tx, ty)[None]
    cov, sh = tor._iso_cov(0.15)[None], np.zeros((1, 1, 3), np.float32)
    G = _falloff(tor._fwd(p, cov, np.array([0.5], np.float32), sh, W, H), 0, x, y)
    assert 0.01 < G < 0.5
    f = tor._fwd(p, cov, np.array([(1 + sign * eps) / 255 / G], np.float32), sh, W, H)
    m = ro.decision_margins(f, W, H)
    assert m.alpha[y, x] == pytest.approx(eps, abs=2e-6)
    assert f.n_contrib[y, x] == (1 if sign > 0 else 0)
    assert m.T[y, x] == (pytest.approx(1 / 1e-4, rel=1e-2) if sign > 0 else ro.NO_MARGIN)   # T (1 - alpha) ~ 1
    assert m.power[y, x] == ro.NO_MARGIN
    unsettled = ~ro.settled_mask(m, DELTA)
    assert unsettled[y, x] == (eps <= DELTA)
    unsettled[y, x] = False
    assert not unsettled.any()
    assert ro.unsettled_kinds(m, DELTA)["alpha"][y, x] == (eps <= DELTA)


@pytest.mark.parametrize("sign", [+1, -1])
@pytest.mark.parametrize("eps", [0.5 * DELTA, 2 * DELTA])
def test_transmittance_margin_of_an_opaque_stack(sign, eps):
    """Three wide Gaussians in depth order with alpha 0.9, 0.95 and 0.98 - 0.02 sign eps at pixel (9, 6): the third
    entry's test is T (1 - alpha) = 0.005 * 0.02 (1 + sign eps) = 1e-4 (1 + sign eps).  It blends iff sign > 0."""
    W = H = 16
    x, y = 9, 6
    _, _, _, tx, ty = tor._identity_camera(W, H)
    means = np.stack([tor._point_for_pixel(8.3, 7.2, 2.0 + 0.5 * k, W, H, tx, ty) for k in range(3)])
    cov, sh = np.stack([tor._iso_cov(1.0)] * 3), np.zeros((3, 1, 3), np.float32)
    f0 = tor._fwd(means, cov, np.full(3, 0.5, np.float32), sh, W, H)
    alphas = [0.9, 0.95, 0.98 - 0.02 * sign * eps]
    opac = np.array([a / _falloff(f0, g, x, y) for g, a in enumerate(alphas)], np.float32)
    f = tor._fwd(means, cov, opac, sh, W, H)
    m = ro.decision_margins(f, W, H)
    # the float32 opacities round alpha by 3e-8, which 1 - alpha magnifies: 1.5e-6 of 0.02, 1.2e-6 of 0.05, ...
    assert m.T[y, x] == pytest.approx(eps, abs=1e-5)
    assert f.n_contrib[y, x] == (3 if sign > 0 else 2)
    assert m.alpha[y, x] > 100 and m.power[y, x] == ro.NO_MARGIN
    unsettled = ~ro.settled_mask(m, DELTA)
    assert unsettled[y, x] == (eps <= DELTA)
    assert ro.unsettled_kinds(m, DELTA)["T"][y, x] == (eps <= DELTA)
    unsettled[y, x] = False
    assert not unsettled.any()


def test_power_margin_of_a_cancelling_conic():
    """Hand-written records: one entry at (5, 5) on a 16x16 tile with the singular conic (1, b, 1).  With b = 1 the
    power -0.5 (dx^2 + dy^2) - dx dy is an exact 0 of cancelling products along dx = -dy, with b one ulp above 1 it is
    positive there: both are on the sign test's threshold.  The centre itself (dx = dy = 0: every product is 0, in any
    order) and every other pixel (power <= -0.5) are not."""
    W = H = 16
    for b in (np.float32(1), np.nextafter(np.float32(1), np.float32(2))):
        pre = ro.Preprocessed(np.ones(1, np.float32), np.ones(1, np.int32), np.array([[5, 5]], np.float32),
                              np.array([[1, b, 1, 0.5]], np.float32), np.ones((1, 3), np.float32),
                              np.zeros((1, 3), np.uint8), np.array([[0, 0, 1, 1]], np.int32), np.ones(1, np.uint32))
        binned = ro.Binned(np.zeros(1, np.uint64), np.zeros(1, np.uint32), np.array([[0, 1]], np.uint32))
        f = ro.Forward(pre, binned, np.zeros((3, H, W), np.float32), np.ones((H, W), np.float32),
                       np.zeros((H, W), np.uint32))
        m = ro.decision_margins(f, W, H)
        ys, xs = np.mgrid[0:H, 0:W]
        line = (xs + ys == 10) & (xs != 5)
        assert np.array_equal(ro.unsettled_kinds(m, DELTA)["power"], line)
        assert np.array_equal(m.power < ro.NO_MARGIN, line)
        assert m.power[6, 4] == (0 if b == 1 else pytest.approx(1.2e-7, rel=0.1))
        assert not ro.settled_mask(m, DELTA)[6, 4] and ro.settled_mask(m, DELTA)[5, 5]


@pytest.mark.parametrize("key", CPU_SCENES)
def test_float32_oracle_is_settled_where_the_mask_says_so(key):
    ref = _ref(key)
    f, f64 = ref.f, ref.f64
    for d in (1e-5, 1e-4, 1e-3):
        kinds = ro.unsettled_kinds(ref.margins, d)
        print(f"UNSETTLED {key} delta={d:g} total={(~ro.settled_mask(ref.margins, d)).mean():.4%} "
              + " ".join(f"{k}={v.mean():.4%}" for k, v in kinds.items()))
    c = ref.counts()
    assert c["unsettled"] <= MAX_UNSETTLED * c["pixels"], c
    ok = ref.settled
    assert np.array_equal(f.n_contrib[ok], f64.n_contrib[ok])
    assert np.abs(f.color - f64.color).max(0)[ok].max() <= util.SETTLED_COLOR_TOL
    assert np.abs(f.final_T - f64.final_T)[ok].max() <= util.SETTLED_T_TOL
    # as a comparison through the helper the GPU test uses: the float64 composite as "got"
    util.compare_settled_forward(ref, f64.color, f64.n_contrib, f64.final_T, tag=f"{key}/float64-on-records")
    g32, g64 = ref.gradients()
    own = {k: util.element_ratio(g32[k], g64[k])[0] for k in g32}
    print(f"OWN_RATIO {key} " + " ".join(f"{k}={v:.4f}" for k, v in own.items()))
    assert max(own.values()) <= OWN_BAR, own
    # a masked pixel contributes exactly nothing: the gradients do not see what dL/dC was there
    if key == "ragged":
        d = np.random.default_rng(1).standard_normal((3, ref.H, ref.W)).astype(np.float32)
        d2 = np.where(ok[None], d, 0).astype(np.float32)
        assert np.array_equal(d2, ref.d_img(1))
        b = util.oracle_backward(f, ref.a, d2, ref.bg, ref.W, ref.H)
        assert np.array_equal(b.dL_dmeans, g32["means"]) and np.array_equal(b.dL_dsh, g32["col"])


def _old_forward_bars(color, n_contrib, final_T, f) -> bool:
    """The composite bars of util.check_forward, restated (check_forward itself runs the GPU)."""
    diff = np.abs(color - f.color)
    return bool(diff.max() <= 1e-2 and (diff <= 2e-5).mean() >= 0.999 and util.psnr(color, f.color) > 60.0
                and (n_contrib.astype(np.int64) == f.n_contrib.astype(np.int64)).mean() >= 0.999
                and np.abs(final_T - f.final_T).max() <= 1e-2)


def _old_gradient_bars(got, ref) -> bool:
    """The float32-oracle bars of util.check_backward over util.grad_errors."""
    r = util.grad_errors(got, ref)
    return r["max"] <= 2e-3 and r["l2"] <= util.L2_BAR and r["q999"] <= 1.0


def test_planted_errors_pass_the_percentile_bars_and_fail_the_settled_ones():
    """The gap, and that it is closed.  "Got" is the float32 oracle's own output of the 256x256 RE10k-like scene with
    (a) 0.05 % of the settled pixels off by 5e-3 and one n_contrib of them off by one, (b) the gradient rows of 0.05 %
    of the Gaussians (rows below 1 % of the tensor's largest entry: a bug need not sit in the largest) off by 3 x
    their element bar.  (At 20 x the bar on that many rows the norm-wise l2 <= 1e-4 bar does notice, at l2 = 4e-4; the
    percentile never does, and on a tenth of the rows neither would.)"""
    ref = _ref("config1")
    f, rng = ref.f, np.random.default_rng(0)
    ys, xs = np.nonzero(ref.settled)
    pick = rng.choice(ys.size, max(1, int(0.0005 * ref.settled.size)), replace=False)
    color, n_contrib = f.color.copy(), f.n_contrib.copy()
    color[:, ys[pick], xs[pick]] += np.float32(5e-3)
    n_contrib[ys[pick[0]], xs[pick[0]]] += 1
    assert _old_forward_bars(f.color, f.n_contrib, f.final_T, f)
    util.compare_settled_forward(ref, f.color, f.n_contrib, f.final_T, tag="clean")
    assert _old_forward_bars(color, n_contrib, f.final_T, f), "the percentile bars were expected to miss this"
    with pytest.raises(AssertionError, match=rf"{pick.size} settled pixels differ"):
        util.compare_settled_forward(ref, color, n_contrib, f.final_T, tag="planted")

    g32, g64 = ref.gradients()
    got = {k: np.array(v, np.float64) for k, v in g32.items()}
    util.compare_settled_gradients(got, g32, g64, tag="clean")
    for k, v in got.items():
        rows = np.abs(v).reshape(v.shape[0], -1).max(1)
        small = np.nonzero((rows > 0) & (rows <= 0.01 * rows.max()))[0]
        hit = rng.choice(small, max(1, int(0.0005 * v.shape[0])), replace=False)
        v[hit] += 3 * (util.GRAD_ATOL_REL * np.abs(g32[k]).max() + util.GRAD_RTOL * np.abs(g32[k][hit]))
        assert _old_gradient_bars(v, g32[k]), (k, "the percentile bars were expected to miss this", util.grad_errors(v, g32[k]))
        with pytest.raises(AssertionError, match="its bar from the float32 oracle"):
            util.compare_settled_gradients({k: v}, g32, g64, tag="planted")
