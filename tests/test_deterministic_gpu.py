"""The rasterizer under torch.use_deterministic_algorithms(True) (include/pixelsplat_b200.h option "deterministic":
fixed-order composite backward and loss epilogue).

  1. Bit-identical repeats: three runs of the same call give the same bits in every output gradient and in the loss
     sums -- every warp-task variant, colour only, the fused loss, and depth with dL/dD.
  2. The same answer as with the flag off: images, radii and depth bit-identical, gradients and loss sums within the
     1e-6 norm-wise bar of float-atomic order.
  3. The oracle bars of tests/util.check_backward hold with the flag on.
  4. A CUDA graph captured with the flag on replays the eager deterministic step bit for bit.
  5. End to end through DecoderSplattingCUDA: forward + MSE + LossDepth + SSIM, and forward_mse with a depth gradient.
  6. The legacy compositor follows torch's convention for an op without a deterministic implementation.
  7. With the flag off again, the library option reads 0 and the workspace is the default one.
"""
import os

import numpy as np
import pytest
import torch

from pixelsplat_b200 import synthetic
from tests import util

pytestmark = pytest.mark.gpu

DEV = util.DEV
WARP_VARIANTS = {"k1": (2, 1, 1), "k1-nohl": (2, 1, 0), "k2": (2, 2, 1), "k2-nohl": (2, 2, 0),
                 "k4": (2, 4, 1), "k4-nohl": (2, 4, 0)}
ROUTES = ("colour", "loss", "depth", "log")
GRADS = ("means", "cov", "opac", "sh", "means2d")


@pytest.fixture
def det():
    """torch's deterministic flag on for the test; the flag, the library option and the cuBLAS workspace setting torch
    asks for under the flag are restored afterwards, also when the test fails."""
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


_CACHE = {}


def _memo(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


# ------------------------------------------------------------------ scenes: S scenes x V views in one call
def _scene(name):
    """(scenes, V, background) of a named workload."""
    if name == "config0":
        return [synthetic.scene_random_frustum(seed=3)], 1, (0.1, 0.2, 0.3)
    if name == "ragged":
        return [synthetic.scene_random_frustum(seed=6, image_hw=(50, 70), num_gaussians=4000,
                                               z_range=(1.0, 4.0))], 1, (0.0, 0.0, 0.0)
    if name == "s2v2":
        return [synthetic.scene_re10k_like(seed=80 + i, image_hw=(128, 128), target_views=2) for i in range(2)], 2, \
            (0.0, 0.1, 0.0)
    assert name == "config1"
    return [synthetic.scene_re10k_like(seed=0)], 1, (0.0, 0.0, 0.0)


def _inputs(name):
    """Device tensors of a workload: Gaussians [S, P, ...], cameras [S*V, ...], a target image and the upstream
    gradients of the colour and depth images (fixed seeds)."""
    def build():
        scs, V, bg = _scene(name)
        S = len(scs)
        H, W = scs[0].image_shape
        args = [[util.view_args(sc, view=v, scale_invariant=False) for v in range(V)] for sc in scs]
        stack = lambda k: torch.stack([args[s][0][k] for s in range(S)]).to(DEV).contiguous()
        cam = lambda k: torch.stack([args[s][v][k] for s in range(S) for v in range(V)]).to(DEV).contiguous()
        g = torch.Generator().manual_seed(11)
        return dict(
            S=S, V=V, H=H, W=W, sh_degree=args[0][0]["sh_degree"],
            means=stack("means"), cov=stack("cov6"), opac=stack("opac"), sh=stack("sh"),
            viewmatrix=cam("vm"), projmatrix=cam("pm"), campos=cam("campos"),
            tanfov=torch.tensor([[args[s][v]["tanfovx"], args[s][v]["tanfovy"]] for s in range(S) for v in range(V)],
                                device=DEV),
            background=torch.tensor([bg] * (S * V), dtype=torch.float32, device=DEV),
            near_far=torch.tensor([[float(sc.near[v]), float(sc.far[v])] for sc in scs for v in range(V)],
                                  dtype=torch.float32, device=DEV),
            target=torch.rand((S * V, 3, H, W), generator=g).to(DEV),
            w_color=torch.randn((S * V, 3, H, W), generator=g).to(DEV),
            w_depth=torch.randn((S * V, H, W), generator=g).to(DEV),
            w_sse=torch.rand((S * V,), generator=g).to(DEV) + 0.5)
    return _memo(("inputs", name), build)


def run(x, route):
    """One forward + backward of `route` ("colour", "loss", or a depth mode) through the public rasterizer entry
    points.  Returns every output (detached) and every input gradient."""
    from pixelsplat_b200.rasterizer import (rasterize_gaussians, rasterize_gaussians_mse,
                                            rasterize_gaussians_with_depth)
    leaves = {k: x[k].clone().requires_grad_(True) for k in ("means", "cov", "opac", "sh")}
    leaves["means2d"] = torch.zeros((x["S"] * x["V"], x["means"].shape[1], 3), device=DEV, requires_grad=True)
    kw = dict(viewmatrix=x["viewmatrix"], projmatrix=x["projmatrix"], campos=x["campos"], tanfov=x["tanfov"],
              background=x["background"], image_shape=(x["H"], x["W"]), views_per_scene=x["V"],
              sh_degree=x["sh_degree"])
    L = [leaves[k] for k in ("means", "cov", "opac", "sh")]
    out = {}
    if route == "colour":
        color, radii = rasterize_gaussians(*L, means2d=leaves["means2d"], **kw)
        loss = (color * x["w_color"]).sum()
    elif route == "loss":
        sse, sse_clipped, color, radii = rasterize_gaussians_mse(*L, x["target"], **kw)
        out.update(sse=sse.detach(), sse_clipped=sse_clipped)
        loss = (sse * x["w_sse"]).sum()
    else:
        color, depth, radii = rasterize_gaussians_with_depth(*L, depth_mode=route, near_far=x["near_far"], **kw)
        out["depth"] = depth.detach()
        loss = (color * x["w_color"]).sum() + (depth * x["w_depth"]).sum()
    loss.backward()
    out.update(color=color.detach(), radii=radii)
    out.update({k: v.grad for k, v in leaves.items() if v.grad is not None})
    return out


def assert_same_bits(a, b, tag):
    assert a.keys() == b.keys(), tag
    for k in a:
        assert torch.equal(a[k], b[k]), (tag, k, float((a[k].double() - b[k].double()).abs().max()))


def _same_up_to_atomic_order(a, b, tag):
    """a == b bit for bit, or norm-wise within 1e-6 (what float-atomic order moves)."""
    if torch.equal(a, b):
        return
    e = float((a.double() - b.double()).norm() / max(float(b.double().norm()), 1e-30))
    assert e <= 1e-6, (tag, e)


# ------------------------------------------------------------------ 1. bit-identical repeats
def _repeats(name, route, n=3):
    x = _inputs(name)
    first = run(x, route)
    assert all(k in first for k in GRADS if not (k == "means2d" and route != "colour")), first.keys()
    for _ in range(n - 1):
        assert_same_bits(run(x, route), first, (name, route))
    return first


@pytest.mark.parametrize("variant", list(WARP_VARIANTS))
@pytest.mark.parametrize("name", ["config0", "ragged"])
def test_repeats_are_bit_identical_per_variant(det, name, variant):
    with util.composite_variant(*WARP_VARIANTS[variant]):
        for route in ROUTES:
            _repeats(name, route)


@pytest.mark.parametrize("name", ["s2v2", "config1"])
def test_repeats_are_bit_identical(det, name):
    """S = 2 x V = 2 at 128x128 and configs[1] (256x256, P = 393 216) with the automatic variant.  Without the
    fixed-order path the configs[1] gradients differ between runs in the last bits."""
    for route in ROUTES:
        _repeats(name, route)


# ------------------------------------------------------------------ 2. the same answer as with the flag off
@pytest.mark.parametrize("name", ["config0", "ragged", "s2v2"])
def test_same_answer_as_flag_off(det, name):
    x = _inputs(name)
    for route in ROUTES:
        on = run(x, route)
        torch.use_deterministic_algorithms(False)
        try:
            off = run(x, route)
        finally:
            torch.use_deterministic_algorithms(True)
        for k in ("color", "radii", "depth"):
            if k in on:
                assert torch.equal(on[k], off[k]), (name, route, k)
        for k in (*GRADS, "sse", "sse_clipped"):
            if k in on:
                _same_up_to_atomic_order(on[k], off[k], (name, route, k))
        if route == "loss":
            # the fixed-order sums against float64 sums of the rendered image (every task's share counts)
            ref = ((on["color"].double() - x["target"].double()) ** 2).sum(dim=(1, 2, 3))
            e = float(((on["sse"].double() - ref).abs() / ref).max())
            assert e <= 1e-5, (name, e)


# ------------------------------------------------------------------ 3. oracle bars with the flag on
def _oracle_scene(name):
    if name == "config0":
        sc = synthetic.scene_random_frustum(seed=3)
        return util.view_args(sc), (0.1, 0.2, 0.3), *sc.image_shape
    sc = synthetic.scene_random_frustum(seed=6, image_hw=(50, 70), num_gaussians=4000, z_range=(1.0, 4.0))
    return util.view_args(sc), (0.0, 0.0, 0.0), 50, 70


@pytest.mark.parametrize("variant", list(WARP_VARIANTS))
@pytest.mark.parametrize("name", ["config0", "ragged"])
def test_oracle_bars_hold(det, name, variant):
    a, bg, H, W = _memo(("oracle_scene", name), lambda: _oracle_scene(name))
    d_img = np.random.default_rng(1).standard_normal((3, H, W)).astype(np.float32)
    refs = _memo(("refs", name), lambda: util.oracle_gradients(a, bg, H, W, d_img))
    with util.composite_variant(*WARP_VARIANTS[variant]):
        util.check_backward(a, bg, H, W, seed=1, refs=refs)


# ------------------------------------------------------------------ 4. CUDA graph
def test_cuda_graph_replay_matches_eager(det):
    from pixelsplat_b200.decoder.cuda_splatting import render_views_with_depth
    sc = synthetic.scene_re10k_like(seed=50, image_hw=(64, 64), target_views=2)
    t = lambda v: v.to(DEV)[None]
    cam = (t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far), (64, 64))
    bg = torch.zeros(1, 2, 3, device=DEV)
    leaves = [t(v).requires_grad_(True) for v in (sc.means, sc.covariances, sc.harmonics, sc.opacities)]
    g = torch.Generator().manual_seed(3)
    w_c, w_d = torch.randn(1, 2, 3, 64, 64, generator=g).to(DEV), torch.randn(1, 2, 64, 64, generator=g).to(DEV)

    def step():
        for l in leaves:
            l.grad = None
        color, depth = render_views_with_depth(*cam, bg, *leaves, mode="depth")
        ((color * w_c).sum() + (depth * w_d).sum()).backward()
        return color.detach(), depth.detach(), [l.grad for l in leaves]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager = step()              # also sizes the binning capacity of this shape
        eager = [eager[0].clone(), eager[1].clone(), [v.clone() for v in eager[2]]]
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])
        for a, b in zip(out[2], eager[2]):
            assert torch.equal(a, b)


# ------------------------------------------------------------------ 5. end to end
def _decoder_inputs():
    from pixelsplat_b200.decoder import DecoderSplattingCUDA, DecoderSplattingCUDACfg
    scs = [synthetic.scene_re10k_like(seed=30 + i, image_hw=(48, 80), target_views=3) for i in range(2)]
    t = lambda k: torch.stack([getattr(sc, k) for sc in scs]).to(DEV)
    dec = DecoderSplattingCUDA(DecoderSplattingCUDACfg("splatting_cuda"),
                               type("D", (), {"background_color": [0.1, 0.2, 0.3]})()).to(DEV)
    target = torch.rand(2, 3, 3, 48, 80, generator=torch.Generator().manual_seed(3)).to(DEV)
    d_dep = torch.randn(2, 3, 48, 80, generator=torch.Generator().manual_seed(5)).to(DEV)
    cam = (t("extrinsics"), t("intrinsics"), t("near"), t("far"), (48, 80))
    return dec, cam, target, d_dep, [t(k) for k in ("means", "covariances", "harmonics", "opacities")]


def test_decoder_training_step_is_bit_identical(det):
    """DecoderSplattingCUDA.forward(depth_mode="depth") -> MSE + LossDepth + (1 - SSIM) of the colour -> backward."""
    from pixelsplat_b200 import loss as L
    from pixelsplat_b200.decoder import Gaussians
    dec, cam, target, _, g0 = _decoder_inputs()
    ld = L.LossDepth(L.LossDepthCfgWrapper(L.LossDepthCfg(0.25, 12.0, True)))
    batch = {"target": {"near": cam[2], "far": cam[3], "image": target}}

    def step():
        leaves = [v.clone().requires_grad_(True) for v in g0]
        out = dec.forward(Gaussians(*leaves), *cam, depth_mode="depth")
        value = ((out.color - target) ** 2).mean() + ld(out, batch) + \
            (1 - L.ssim(target.flatten(0, 1), out.color.flatten(0, 1))).mean()
        value.backward()
        return [value.detach(), out.color.detach(), out.depth.detach()] + [v.grad for v in leaves]

    a, b = step(), step()
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), i


def test_forward_mse_with_depth_is_bit_identical(det):
    """forward_mse(depth_mode="depth"): the fused loss epilogue and a depth gradient in one pass."""
    from pixelsplat_b200.decoder import Gaussians
    dec, cam, target, d_dep, g0 = _decoder_inputs()

    def step():
        leaves = [v.clone().requires_grad_(True) for v in g0]
        out, sse, sse_clipped = dec.forward_mse(Gaussians(*leaves), *cam, target, depth_mode="depth")
        (sse.sum() + (out.depth * d_dep).sum()).backward()
        return [sse.detach(), sse_clipped, out.depth.detach()] + [v.grad for v in leaves]

    a, b = step(), step()
    for i, (u, v) in enumerate(zip(a, b)):
        assert torch.equal(u, v), i


# ------------------------------------------------------------------ 6. the legacy compositor
def test_legacy_compositor_alerts(det):
    x = _inputs("config0")
    with util.composite_variant(1, 1, 0):
        with pytest.raises(RuntimeError, match="does not have a deterministic implementation"):
            run(x, "colour")
        torch.use_deterministic_algorithms(True, warn_only=True)
        with pytest.warns(UserWarning, match="does not have a deterministic implementation"):
            out = run(x, "colour")
    assert torch.isfinite(out["color"]).all() and out["means"].abs().sum() > 0


# ------------------------------------------------------------------ 7. flag off again
def test_flag_off_restores_the_default_mode():
    from pixelsplat_b200 import _lib
    assert not torch.are_deterministic_algorithms_enabled()
    x = _inputs("config0")
    run(x, "loss")
    assert _lib.get_option("deterministic") == 0
    d = _lib.RasterDesc(1, 1, x["means"].shape[1], 16, 3, 0, 0, 64, 64, 0, 0, 100000, 0, 0)
    vp = x["means"].shape[1]
    align = lambda n: (n + 255) // 256 * 256
    assert _lib.sizes(d).backward_bytes == align(vp * 8) + 2 * align(vp * 16)
