"""The CUDA rasterizer against the oracle with no anonymous allowance (tests/util.py, "settled pixels").

The other parity tests forgive 0.1 % (or 0.5 %) of the pixels and the top 0.1 % of the gradient entries, whichever they
are.  Here the oracle names the pixels it forgives: those with a decision (alpha vs 1/255, T (1 - alpha) vs 1e-4, the
sign of power) within util.SETTLED_DELTA of its threshold.  Per view:
  * forward: front end bit-exact; on EVERY other pixel n_contrib equal, |colour| <= 2e-5, |final_T| <= 1e-5; a wrong
    pixel that is not unsettled fails with its coordinates, tile, list length and n_contrib on both sides;
  * backward: dL/dC seeded, zero on the unsettled pixels; EVERY entry of the means, covariance, opacity, SH / colour
    and means2d gradients within the mixed element bar |d| / (1e-5 max|ref| + 1e-3 |ref|) <= 1 of the float32 oracle,
    and within max(1, 2 x the float32 oracle's own ratio) of the float64 composite on the float32 records.
Each line SETTLED_FWD / SETTLED_BWD of the output (-s) lists the unsettled count by kind of decision, how many of those
the GPU really decided differently, the worst settled-pixel errors and the worst gradient ratio per tensor.

Scenes are the ones whose paths can go wrong on a few pixels only: ragged tiles, early termination, lists far past one
run and past the live-list limit, equal depths, every compositor variant, both tile sorts, the fixed-order backward,
several views per call, 256x256 and 512x512 RE10k-like scenes."""
import os

import numpy as np
import pytest
import torch

from pixelsplat_b200 import synthetic
from tests import util

pytestmark = pytest.mark.gpu

# name -> (composite_impl, composite_segments, composite_hit_lists); "auto" is what an unforced call selects
VARIANTS = {"auto": (2, 0, 2), "legacy": (1, 1, 0),
            "k1": (2, 1, 1), "k1-nohl": (2, 1, 0), "k2": (2, 2, 1), "k2-nohl": (2, 2, 0),
            "k4": (2, 4, 1), "k4-nohl": (2, 4, 0)}
MAX_UNSETTLED = 0.03      # of a view's pixels: the mask must not grow into an allowance of its own (measured: up to
                          # 0.8 % at 256x256, 2.1 % at 512x512 where a pixel walks ~4000 entries)


def _frustum(bg=(0.0, 0.0, 0.0), use_sh=True, **kw):
    sc = synthetic.scene_random_frustum(**kw)
    return util.view_args(sc, use_sh=use_sh), bg, *sc.image_shape


def _ties():
    sc = synthetic.scene_random_frustum(seed=13, image_hw=(32, 32), num_gaussians=900)
    sc.means[:, 2] = 3.0
    sc.means[:300, 2] = 5.0
    return util.view_args(sc), (0.0, 0.0, 0.0), 32, 32


def _re10k(**kw):
    sc = synthetic.scene_re10k_like(**kw)
    return util.view_args(sc), (0.0, 0.0, 0.0), *sc.image_shape


SCENES = {
    "config0": lambda: _frustum(seed=3),
    "config0-bg": lambda: _frustum((0.1, 0.2, 0.3), seed=3),
    **{f"sh{d}": (lambda d=d: _frustum(seed=4, sh_degree=d)) for d in range(4)},
    "colors-precomp": lambda: _frustum((0.2, 0.0, 0.1), use_sh=False, seed=5, sh_degree=0),
    "ragged": lambda: _frustum(seed=6, image_hw=(50, 70), num_gaussians=4000, z_range=(1.0, 4.0)),
    "long16": lambda: _frustum(seed=7, image_hw=(16, 16), num_gaussians=30000, z_range=(2.0, 30.0)),
    "long32": lambda: _frustum(seed=8, image_hw=(32, 32), num_gaussians=14000, z_range=(2.0, 30.0)),
    "ties": _ties,
    "config1": lambda: _re10k(seed=0),
    "config4": lambda: _re10k(seed=1, image_hw=(512, 512), context_views=3),
}
_REFS = {}


def _ref(key) -> util.SettledRef:
    """The oracle side of a scene, computed once per module and shared by the variant sweeps."""
    if key not in _REFS:
        _REFS[key] = util.SettledRef(*SCENES[key]())
        c = _REFS[key].counts()
        assert c["unsettled"] <= MAX_UNSETTLED * c["pixels"], (key, c)
    return _REFS[key]


def _check(key, variant="auto", sort_impl=0, backward=True):
    ref, tag = _ref(key), f"{key}/{variant}/sort{sort_impl}"
    with util.composite_variant(*VARIANTS[variant]):
        util.check_forward_settled(ref, sort_impl=sort_impl, tag=tag)
        if backward:
            util.check_backward_settled(ref, tag=tag)


@pytest.mark.parametrize("key", list(SCENES))
def test_every_scene(key):
    """Forward and backward of every scene through the variant an unforced call selects."""
    _check(key)
    f = _ref(key).f
    count = f.binned.ranges[:, 1] - f.binned.ranges[:, 0]
    if key == "ragged":
        assert (f.final_T < 1e-3).mean() > 0.05                       # early termination on many pixels
    if key == "long16":
        assert count.max() > 12288                                    # past the shared-memory sorts
    if key == "long32":
        assert count.max() > 2048


@pytest.mark.parametrize("key", ["config0", "ragged", "long16", "long32", "ties"])
def test_second_tile_sort(key):
    _check(key, sort_impl=1, backward=False)


@pytest.mark.parametrize("variant", [v for v in VARIANTS if v != "auto"])
@pytest.mark.parametrize("key", ["config0-bg", "ragged", "long16", "ties"])
def test_every_variant(key, variant):
    """List runs K = 1, 2, 4 with and without hit lists, and the legacy compositor."""
    _check(key, variant)


@pytest.mark.parametrize("variant", ["k1", "k2", "k2-nohl", "k4", "legacy"])
def test_config1_variants(variant):
    _check("config1", variant)


@pytest.fixture
def det():
    """torch's deterministic flag (the fixed-order composite backward) on for the test, restored afterwards."""
    from pixelsplat_b200 import _lib
    flag, warn_only = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    cublas = os.environ.get("CUBLAS_WORKSPACE_CONFIG")
    os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(flag, warn_only=warn_only)
        _lib.set_option("deterministic", 0)
        if cublas is None:
            os.environ.pop("CUBLAS_WORKSPACE_CONFIG", None)
        else:
            os.environ["CUBLAS_WORKSPACE_CONFIG"] = cublas


@pytest.mark.parametrize("variant", ["auto", "k1", "k2-nohl", "k4"])
@pytest.mark.parametrize("key", ["config0-bg", "ragged", "long16", "config1"])
def test_fixed_order_backward(det, key, variant):
    ref, tag = _ref(key), f"{key}/{variant}/det"
    with util.composite_variant(*VARIANTS[variant]):
        util.check_backward_settled(ref, tag=tag)


def test_batched_scenes_and_views():
    """S = 2 scenes x V = 4 views at 256x256 in one rasterize_gaussians call, with the oracle's host-side cameras so
    that the front end stays bit-exact (render_views computes its cameras on the device, which moves the per-Gaussian
    records by an ulp and with them the lists).  Every view against its own settled mask; dL/dC zero on each view's
    unsettled pixels; each scene's gradients against the view sums of the oracle's."""
    from concurrent.futures import ThreadPoolExecutor

    from tests.test_composite_variants_gpu import _batched
    S, V, H, W = 2, 4, 256, 256
    scs = [synthetic.scene_re10k_like(seed=60 + i, image_hw=(H, W), target_views=V) for i in range(S)]

    def job(sv):
        s, v = sv
        ref = util.SettledRef(util.view_args(scs[s], view=v, scale_invariant=False), (0.0, 0.0, 0.0), H, W)
        ref.gradients(seed=5 + s * V + v)
        return ref

    with ThreadPoolExecutor(8) as ex:          # the C oracle releases the GIL
        refs = list(ex.map(job, [(s, v) for s in range(S) for v in range(V)]))
    d_img = np.stack([refs[i].d_img(seed=5 + i) for i in range(S * V)]).reshape(S, V, 3, H, W)
    color, st, grads, _ = _batched(scs, V, H, W, d_img)
    im = st.intermediates()
    n_contrib, final_T = im["n_contrib"].cpu().numpy(), im["final_T"].cpu().numpy()
    for i, ref in enumerate(refs):
        c = ref.counts()
        assert c["unsettled"] <= MAX_UNSETTLED * c["pixels"], (i, c)
        util.compare_settled_forward(ref, color[i // V, i % V], n_contrib[i], final_T[i], tag=f"s2v4/view{i}")
    for s in range(S):
        sums = [{k: sum(refs[s * V + v].gradients(5 + s * V + v)[j][k] for v in range(V))
                 for k in ("means", "cov", "opac", "col")} for j in (0, 1)]
        util.compare_settled_gradients(grads[s], *sums, tag=f"s2v4/scene{s}")
