"""The rasterizer backward writes every element of every output gradient (the autograd path allocates them with
torch.empty): each call below hands ps_raster_backward gradient buffers and scratch filled with NaN, and checks
that every element comes back finite, that it equals what the same call returns into zero-filled buffers (bit for
bit in deterministic mode), and that the elements that take no gradient are exactly zero:
  * Gaussians on screen in no view of their scene (all of their rows), and every Gaussian after a binning overflow;
  * the lower triangle of a 3x3 covariance, SH coefficients above sh_degree, the third lane of d_means2d.
Covered: 3x3 and triu covariances, SH layouts M3 and 3M, the e3nn basis, precomputed colours (M = 0), S > 1 scenes
with V > 1 views, a depth gradient, the legacy compositor, an overflowing capacity and a scene with nothing on
screen.  A single-view call is also held to the float32 oracle.
"""
import contextlib
import ctypes

import pytest
import torch

from pixelsplat_b200 import _lib, synthetic
from tests import util

pytestmark = pytest.mark.gpu

DEV = util.DEV


@contextlib.contextmanager
def _deterministic(on):
    _lib.set_option("deterministic", 1 if on else 0)
    try:
        yield
    finally:
        _lib.set_option("deterministic", 0)


def _inputs(scs, V, sh_degree=None, cov3x3=False, sh_layout=_lib.PS_SH_M3, use_sh=True, behind=False):
    """Device inputs of S scenes x V views (each scene's Gaussians shared by its views), unscaled cameras."""
    S = len(scs)
    H, W = scs[0].image_shape
    args = [[util.view_args(sc, view=v, scale_invariant=False, use_sh=use_sh) for v in range(V)] for sc in scs]
    stack = lambda k: torch.stack([args[s][0][k] for s in range(S)]).to(DEV).contiguous()
    cam = lambda k: torch.stack([args[s][v][k] for s in range(S) for v in range(V)]).to(DEV).contiguous()
    means, cov6, opac = stack("means"), stack("cov6"), stack("opac")
    if behind:                                         # every Gaussian 5 units behind the (single) camera
        assert S * V == 1
        vm = cam("vm")[0]                              # column-major: view-space z = vm[2, 6, 10] . p + vm[14]
        means = (cam("campos")[0] - 5.0 * vm[[2, 6, 10]]).expand_as(means).contiguous()
    if cov3x3:
        i = torch.tensor([[0, 1, 2], [1, 3, 4], [2, 4, 5]], device=DEV)
        cov = cov6[..., i].contiguous()
    else:
        cov = cov6
    if use_sh:
        sh = stack("sh")                               # [S, P, M, 3]
        if sh_layout == _lib.PS_SH_3M:
            sh = sh.transpose(-1, -2).contiguous()
        M = sh.shape[2] if sh_layout == _lib.PS_SH_M3 else sh.shape[3]
    else:
        sh, M = stack("colors"), 0
    g = torch.Generator().manual_seed(5)
    return dict(S=S, V=V, P=means.shape[1], M=M, H=H, W=W, sh_layout=sh_layout,
                deg=args[0][0]["sh_degree"] if sh_degree is None else sh_degree, cov3x3=cov3x3,
                means=means, cov=cov, opac=opac, sh=sh, vm=cam("vm"), pm=cam("pm"), campos=cam("campos"),
                tanfov=torch.tensor([[args[s][v]["tanfovx"], args[s][v]["tanfovy"]] for s in range(S) for v in range(V)],
                                    dtype=torch.float32, device=DEV),
                bg=torch.full((S * V, 3), 0.1, device=DEV),
                near_far=torch.tensor([[float(sc.near[v]), float(sc.far[v])] for sc in scs for v in range(V)],
                                      dtype=torch.float32, device=DEV),
                d_color=torch.randn((S * V, 3, H, W), generator=g).to(DEV),
                d_depth=torch.randn((S * V, H, W), generator=g).to(DEV))


def _run(x, capacity=None, depth_mode=0, basis=_lib.PS_SH_BASIS_3DGS):
    """Forward, then two backwards of the same forward state: into NaN-filled and into zero-filled buffers.
    Returns (radii [S*V, P], instance count, NaN-filled gradients, zero-filled gradients)."""
    S, V, P, H, W = x["S"], x["V"], x["P"], x["H"], x["W"]
    cap = capacity if capacity is not None else 64 * S * V * P + 4096
    desc = _lib.RasterDesc(S, V, P, x["M"], x["deg"], x["sh_layout"],
                           _lib.PS_COV_3X3 if x["cov3x3"] else _lib.PS_COV_TRIU6, H, W, 0, 0, cap, basis, depth_mode)
    sz = _lib.sizes(desc)
    geom = torch.empty(sz.geom_bytes, dtype=torch.uint8, device=DEV)
    binning = torch.empty(sz.binning_bytes, dtype=torch.uint8, device=DEV)
    image = torch.empty(sz.image_bytes, dtype=torch.uint8, device=DEV)
    state = _lib.RasterState(geom.data_ptr(), geom.numel(), binning.data_ptr(), binning.numel(),
                             image.data_ptr(), image.numel())
    inputs = _lib.RasterInputs(x["means"].data_ptr(), x["cov"].data_ptr(), x["opac"].data_ptr(), x["sh"].data_ptr(),
                               x["vm"].data_ptr(), x["pm"].data_ptr(), x["campos"].data_ptr(), x["tanfov"].data_ptr(),
                               x["bg"].data_ptr(), None, x["near_far"].data_ptr())
    color = torch.empty((S * V, 3, H, W), device=DEV)
    radii = torch.empty((S * V, P), dtype=torch.int32, device=DEV)
    n_host = torch.zeros(2, dtype=torch.int64).pin_memory()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.lib.ps_raster_forward(ctypes.byref(desc), ctypes.byref(inputs), ctypes.byref(state),
                                          ctypes.c_void_p(color.data_ptr()), ctypes.c_void_p(radii.data_ptr()),
                                          ctypes.c_void_p(n_host.data_ptr()), stream), "ps_raster_forward")
    torch.cuda.synchronize()

    def backward(fill):
        grads = dict(means=torch.full_like(x["means"], fill), cov=torch.full_like(x["cov"], fill),
                     opac=torch.full_like(x["opac"], fill), sh=torch.full_like(x["sh"], fill),
                     m2d=torch.full((S * V, P, 3), fill, device=DEV))
        scratch = torch.full((sz.backward_bytes,), 0xFF if fill != 0 else 0, dtype=torch.uint8, device=DEV)
        rg = _lib.RasterGrads(*(grads[k].data_ptr() for k in ("means", "cov", "opac", "sh", "m2d")))
        common = (ctypes.byref(desc), ctypes.byref(inputs), ctypes.byref(state))
        tail = (ctypes.c_void_p(scratch.data_ptr()), scratch.numel(), ctypes.byref(rg), stream)
        if depth_mode:
            rc = _lib.lib.ps_raster_backward_depth(*common, ctypes.c_void_p(x["d_color"].data_ptr()), None, None,
                                                   ctypes.c_void_p(x["d_depth"].data_ptr()), *tail)
        else:
            rc = _lib.lib.ps_raster_backward(*common, ctypes.c_void_p(x["d_color"].data_ptr()), *tail)
        _lib.check(rc, "ps_raster_backward")
        torch.cuda.synchronize()
        return grads

    return radii, int(n_host[0]), backward(float("nan")), backward(0.0)


def _check(x, radii, nan_g, zero_g, exact, all_zero=False):
    S, V, P = x["S"], x["V"], x["P"]
    for k in nan_g:
        a, b = nan_g[k], zero_g[k]
        assert torch.isfinite(a).all(), (k, int((~torch.isfinite(a)).sum()))
        if exact:
            assert torch.equal(a, b), k
        elif not torch.equal(a, b):
            e = float((a.double() - b.double()).norm() / max(float(b.double().norm()), 1e-30))
            assert e <= 1e-6, (k, e)
    on = (radii.reshape(S, V, P) > 0)
    off = ~on.any(dim=1)                               # [S, P]: on screen in no view of the scene
    if all_zero:
        off = torch.ones_like(off)
        on = torch.zeros_like(on)
    for k in ("means", "cov", "opac", "sh"):
        rows = nan_g[k][off]
        assert torch.equal(rows, torch.zeros_like(rows)), k
    m2d = nan_g["m2d"].reshape(S, V, P, 3)
    assert torch.equal(m2d[..., 2], torch.zeros_like(m2d[..., 2]))
    assert torch.equal(m2d[~on], torch.zeros_like(m2d[~on]))
    if x["cov3x3"]:
        low = nan_g["cov"][..., [1, 2, 2], [0, 0, 1]]
        assert torch.equal(low, torch.zeros_like(low))
    nb = (x["deg"] + 1) ** 2
    if x["M"] > nb:
        sh = nan_g["sh"] if x["sh_layout"] == _lib.PS_SH_M3 else nan_g["sh"].transpose(-1, -2)
        assert torch.equal(sh[:, :, nb:], torch.zeros_like(sh[:, :, nb:]))
    if not all_zero:
        assert float(nan_g["sh"][~off].abs().sum()) > 0 and float(nan_g["means"][~off].abs().sum()) > 0


def _config0():
    return [synthetic.scene_random_frustum(seed=3)]


def _s2v2():
    return [synthetic.scene_re10k_like(seed=80 + i, image_hw=(64, 64), target_views=2) for i in range(2)]


CASES = {
    # name: (scenes, V, _inputs keywords, _run keywords)
    "config0-3x3": (_config0, 1, dict(cov3x3=True), {}),
    "config0-3M-deg1": (_config0, 1, dict(sh_layout=_lib.PS_SH_3M, sh_degree=1), {}),
    "config0-colours": (_config0, 1, dict(use_sh=False), {}),
    "config0-e3nn": (_config0, 1, {}, dict(basis=_lib.PS_SH_BASIS_E3NN)),
    "s2v2-triu-deg2": (_s2v2, 2, dict(sh_degree=2), {}),
    "s2v2-3x3-depth": (_s2v2, 2, dict(cov3x3=True), dict(depth_mode=1)),
}


@pytest.mark.parametrize("det", [False, True], ids=["atomic", "deterministic"])
@pytest.mark.parametrize("name", list(CASES))
def test_every_gradient_element_is_written(name, det):
    scenes, V, kin, krun = CASES[name]
    x = _inputs(scenes(), V, **kin)
    with _deterministic(det):
        radii, n, nan_g, zero_g = _run(x, **krun)
    assert 0 < n
    _check(x, radii, nan_g, zero_g, exact=det)


def test_legacy_compositor_rows():
    x = _inputs(_s2v2(), 2, cov3x3=True, sh_degree=2)
    with util.composite_variant(1):
        radii, _, nan_g, zero_g = _run(x)
    _check(x, radii, nan_g, zero_g, exact=False)


@pytest.mark.parametrize("det", [False, True], ids=["atomic", "deterministic"])
def test_overflow_gives_zero_gradients(det):
    x = _inputs(_s2v2(), 2, cov3x3=True)
    with _deterministic(det):
        radii, n, nan_g, zero_g = _run(x, capacity=64)
    assert n > 64
    _check(x, radii, nan_g, zero_g, exact=True, all_zero=True)


def test_nothing_on_screen_gives_zero_gradients():
    x = _inputs(_config0(), 1, cov3x3=True, behind=True)
    radii, n, nan_g, zero_g = _run(x)
    assert n == 0 and int((radii > 0).sum()) == 0
    _check(x, radii, nan_g, zero_g, exact=True, all_zero=True)


def test_single_view_matches_the_oracle():
    sc = _config0()[0]
    a = util.view_args(sc, scale_invariant=False)
    x = _inputs([sc], 1, cov3x3=True)
    H, W = x["H"], x["W"]
    radii, _, nan_g, _ = _run(x)
    ref32, _ = util.oracle_gradients(a, (0.1, 0.1, 0.1), H, W, x["d_color"][0].cpu().numpy(), with_f64=False)
    iu = ([0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2])
    got = dict(means=nan_g["means"][0], cov=nan_g["cov"][0][:, iu[0], iu[1]], opac=nan_g["opac"][0],
               col=nan_g["sh"][0], m2d=nan_g["m2d"][0, :, :2])
    for k, v in got.items():
        r = util.grad_errors(v.cpu().numpy(), ref32[k])
        assert r["l2"] <= util.L2_BAR and r["q999"] <= 1.0, (k, r)
