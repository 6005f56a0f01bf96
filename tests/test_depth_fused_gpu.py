"""The depth channel of the warp-task compositor (include/pixelsplat_b200.h depth_mode) on the GPU.

  1. Nothing else changes: colour, radii, final_T, n_contrib, run_state, the colour-only gradients and the fused
     loss sums are the same with the depth channel on as off, under every warp-task variant.
  2. The depth image against the oracle rendering the per-Gaussian depth value as the red channel (what
     render_depth_cuda does), every mode, scale_invariant on and off, and against render_depth_views.
  3. Gradients against the oracle decomposition: colour backward + depth-as-colour backward + the depth value's
     chain to the means, every mode under every warp-task variant.
  4. The fused-loss route (forward_mse) with a depth gradient against the unfused route.
  5. A LossDepth step: the fused route and today's two-pass route given the same dL/dD.
  6. CUDA-graph replay, and the legacy compositor (no depth channel: PS_ERR_UNSUPPORTED / two-pass fallback).
"""
import ctypes

import numpy as np
import pytest
import torch

from pixelsplat_b200 import synthetic
from tests import util

pytestmark = pytest.mark.gpu

DEV = util.DEV
MODES = ("depth", "disparity", "relative_disparity", "log")
WARP_VARIANTS = {"k1": (2, 1, 1), "k1-nohl": (2, 1, 0), "k2": (2, 2, 1), "k2-nohl": (2, 2, 0),
                 "k4": (2, 4, 1), "k4-nohl": (2, 4, 0)}


@pytest.fixture(scope="module")
def cache():
    return {}


def _memo(cache, key, fn):
    if key not in cache:
        cache[key] = fn()
    return cache[key]


# ------------------------------------------------------------------ scenes and arguments
def _config0():
    return synthetic.scene_random_frustum(seed=3), (0.1, 0.2, 0.3)


def _re10k64():
    return synthetic.scene_re10k_like(seed=21, image_hw=(64, 64)), (0.0, 0.0, 0.0)


def _ragged():
    return synthetic.scene_random_frustum(seed=6, image_hw=(50, 70), num_gaussians=4000, z_range=(1.0, 4.0)), \
        (0.0, 0.0, 0.0)


def _args(sc, bg, si, view=0):
    """(oracle arguments (rescaled when si), native arguments (un-rescaled Gaussians + scene_scale), scale)."""
    a = util.view_args(sc, view=view, scale_invariant=si)
    near = torch.as_tensor(sc.near[view], dtype=torch.float32)
    scale = (1 / near) if si else torch.tensor(1.0)
    row, col = torch.triu_indices(3, 3)
    n = dict(means=sc.means.float() if si else a["means"], cov6=sc.covariances.float()[:, row, col].contiguous()
             if si else a["cov6"], opac=a["opac"], sh=a["sh"], vm=a["vm"], pm=a["pm"], campos=a["campos"],
             tanfov=(a["tanfovx"], a["tanfovy"]), bg=bg, sh_degree=a["sh_degree"],
             scene_scale=scale.reshape(1) if si else None,
             near_far=torch.stack([sc.near[view], sc.far[view]]).float().reshape(1, 2), H=sc.image_shape[0],
             W=sc.image_shape[1])
    return a, n, float(scale)


def _depth_values(sc, mode, view=0, dtype=torch.float32):
    """d per Gaussian, computed as the reference does: camera-space z from inv(extrinsics) and the un-rescaled
    means (float32), then the mode's transform (pixelsplat_b200.decoder.cuda_splatting.depth_colors)."""
    from pixelsplat_b200.decoder.cuda_splatting import depth_colors
    e = sc.extrinsics[view][None, None].to(dtype)
    return depth_colors(e, sc.means[None].to(dtype), sc.near[view].reshape(1, 1).to(dtype),
                        sc.far[view].reshape(1, 1).to(dtype), mode)[0, 0]


def _chain(sc, mode, view=0):
    """dd/dmean [P, 3] in float64: f'(z) times row 2 of inv(extrinsics) (torch's minimum / maximum rule in log)."""
    e = sc.extrinsics[view].double()
    w2c = torch.linalg.inv(e)
    z = sc.means.double() @ w2c[2, :3] + w2c[2, 3]
    near, far = float(sc.near[view]), float(sc.far[view])
    eps = 1e-10
    if mode == "depth":
        fp = torch.ones_like(z)
    elif mode == "disparity":
        fp = -1 / z ** 2
    elif mode == "relative_disparity":
        fp = (1 / (z + eps) ** 2) / (1 / (near + eps) - 1 / (far + eps) + eps)
    else:
        m = z.clamp(max=near)
        gm = torch.where(z < near, 1.0, torch.where(z == near, 0.5, 0.0))
        gr = torch.where(m > far, 1.0, torch.where(m == far, 0.5, 0.0))
        fp = gm * gr / torch.maximum(m, torch.tensor(far, dtype=torch.float64))
    return (fp[:, None] * w2c[2, :3][None]).numpy()


def native(n, mode=None, d_img=None, d_dep=None, target=None, states=None):
    """One view through rasterize_gaussians_with_depth (mode given) or rasterize_gaussians / _mse (mode None).
    Returns dict(color, depth, radii, sse, sse_clipped, grads)."""
    from pixelsplat_b200.rasterizer import (rasterize_gaussians, rasterize_gaussians_mse,
                                            rasterize_gaussians_with_depth)
    t = lambda x: x.to(DEV)
    leaves = dict(means=t(n["means"])[None].clone().requires_grad_(True),
                  cov=t(n["cov6"])[None].clone().requires_grad_(True),
                  opac=t(n["opac"])[None].clone().requires_grad_(True),
                  col=t(n["sh"])[None].clone().requires_grad_(True))
    kw = dict(viewmatrix=t(n["vm"])[None], projmatrix=t(n["pm"])[None], campos=t(n["campos"])[None],
              tanfov=torch.tensor([n["tanfov"]], device=DEV),
              background=torch.tensor([n["bg"]], dtype=torch.float32, device=DEV), image_shape=(n["H"], n["W"]),
              views_per_scene=1, sh_degree=n["sh_degree"],
              scene_scale=None if n["scene_scale"] is None else t(n["scene_scale"]),
              state_out=states if states is not None else [])
    L = list(leaves.values())
    out = dict(depth=None, sse=None, sse_clipped=None, grads=None)
    tgt = None if target is None else t(target)[None]
    if mode is None and tgt is None:
        out["color"], out["radii"] = rasterize_gaussians(*L, **kw)
    elif mode is None:
        out["sse"], out["sse_clipped"], out["color"], out["radii"] = rasterize_gaussians_mse(*L, tgt, **kw)
    elif tgt is None:
        out["color"], out["depth"], out["radii"] = rasterize_gaussians_with_depth(
            *L, depth_mode=mode, near_far=t(n["near_far"]), **kw)
    else:
        out["sse"], out["sse_clipped"], out["color"], out["depth"], out["radii"] = rasterize_gaussians_with_depth(
            *L, depth_mode=mode, near_far=t(n["near_far"]), target=tgt, **kw)
    loss = None
    if d_img is not None:
        loss = (out["color"] * t(torch.as_tensor(d_img))[None]).sum()
    if tgt is not None and d_img is None:
        loss = out["sse"].sum()
    if d_dep is not None:
        dl = (out["depth"] * t(torch.as_tensor(d_dep))[None]).sum()
        loss = dl if loss is None else loss + dl
    if loss is not None:
        loss.backward()
        out["grads"] = {k: v.grad[0] for k, v in leaves.items()}
    return out


def _depth_oracle_args(a, sc, mode, view=0):
    d = _depth_values(sc, mode, view)
    colors = torch.stack([d, torch.zeros_like(d), torch.zeros_like(d)], -1).contiguous()
    return dict(a, sh=None, colors=colors, sh_degree=0)


def _image_bar(got, ref):
    """DESIGN section 6 image bars, scaled by max(1, max|ref|)."""
    s = max(1.0, float(np.abs(ref).max()))
    diff = np.abs(got - ref) / s
    assert diff.max() <= 1e-2, diff.max()
    assert (diff <= 2e-5).mean() >= 0.999, (diff <= 2e-5).mean()
    return float(diff.max())


# ------------------------------------------------------------------ 1. nothing else changes
def _same_up_to_atomic_order(a, b):
    """a == b bit for bit, or norm-wise within 1e-6: the backward sums per-(view, Gaussian) gradients and the loss
    epilogue its per-view sums with float atomics whose order changes from run to run, so two runs of the SAME
    colour-only call already differ in the last bits.  (The kernels and their inputs are the colour-only ones.)"""
    if torch.equal(a, b):
        return
    e = float((a.double() - b.double()).norm() / max(float(b.double().norm()), 1e-30))
    assert e <= 1e-6, e


@pytest.mark.parametrize("name", list(WARP_VARIANTS))
def test_nothing_else_changes(name):
    for sc, bg in (_config0(), _ragged()):
        _, n, _ = _args(sc, bg, True)
        H, W = n["H"], n["W"]
        d_img = np.random.default_rng(2).standard_normal((3, H, W)).astype(np.float32)
        target = torch.rand(3, H, W, generator=torch.Generator().manual_seed(4))
        with util.composite_variant(*WARP_VARIANTS[name]):
            s0, s1 = [], []
            off = native(n, None, d_img, states=s0)
            on = native(n, "depth", d_img, states=s1)
            i0, i1 = s0[0].intermediates(), s1[0].intermediates()
            K = WARP_VARIANTS[name][1]
            i0["run_state"], i1["run_state"] = i0["run_state"][:, :K - 1], i1["run_state"][:, :K - 1]   # slots written
            for k in ("final_T", "n_contrib", "run_state", "color"):
                assert torch.equal(i0[k], i1[k]), k
            assert torch.equal(off["color"], on["color"]) and torch.equal(off["radii"], on["radii"])
            assert i0["depth_image"] is None and i1["depth_image"] is not None
            for k in off["grads"]:
                _same_up_to_atomic_order(on["grads"][k], off["grads"][k])
            lo, ld = native(n, None, target=target), native(n, "depth", target=target)
            for k in ("sse", "sse_clipped"):
                _same_up_to_atomic_order(ld[k].detach(), lo[k].detach())
            for k in lo["grads"]:
                _same_up_to_atomic_order(ld["grads"][k], lo["grads"][k])


# ------------------------------------------------------------------ 2. depth forward against the oracle
def _check_depth_forward(cache, key, sc, bg, si, modes=MODES, view=0):
    a, n, _ = _args(sc, bg, si, view)
    errs = {}
    for mode in modes:
        ad = _depth_oracle_args(a, sc, mode, view)
        f = _memo(cache, ("dfwd", key, si, mode), lambda: util.oracle_forward(ad, (0, 0, 0), n["W"], n["H"]))
        got = native(n, mode)["depth"][0].detach().cpu().numpy()
        errs[mode] = _image_bar(got, f.color[0])
        assert np.abs(f.color[1:]).max() == 0
    print("DEPTH_FWD", key, si, {k: f"{v:.1e}" for k, v in errs.items()})
    return errs


@pytest.mark.parametrize("si", [True, False])
def test_depth_forward_config0_re10k_ragged(cache, si):
    for key, (sc, bg) in (("config0", _config0()), ("re10k64", _re10k64()), ("ragged", _ragged())):
        _check_depth_forward(cache, key, sc, bg, si)


@pytest.mark.parametrize("name", ["k2", "k4"])
def test_depth_forward_ragged_replays(cache, name):
    """The ragged saturating scene with forced list runs: its replay band exercises the K = 2 / 4 replays."""
    sc, bg = _ragged()
    with util.composite_variant(*WARP_VARIANTS[name]):
        _check_depth_forward(cache, "ragged", sc, bg, True)


def test_depth_forward_batched_views():
    """S = 2 scenes x V = 2 views in one call through render_views_with_depth, every mode, against the oracle per
    view and against today's render_depth_views; the colour equals render_views'."""
    from pixelsplat_b200.decoder.cuda_splatting import render_depth_views, render_views, render_views_with_depth
    scs = [synthetic.scene_re10k_like(seed=80 + i, image_hw=(64, 64), target_views=2) for i in range(2)]
    t = lambda k: torch.stack([getattr(sc, k) for sc in scs]).to(DEV)
    cam = (t("extrinsics"), t("intrinsics"), t("near"), t("far"), (64, 64))
    g = (t("means"), t("covariances"), t("harmonics"), t("opacities"))
    bg = torch.zeros(2, 2, 3, device=DEV)
    with torch.no_grad():
        ref_color = render_views(*cam, bg, *g)
        for mode in MODES:
            color, depth = render_views_with_depth(*cam, bg, *g, mode=mode)
            assert torch.equal(color, ref_color)
            two = render_depth_views(*cam, g[0], g[1], g[3], mode=mode)
            for s in range(2):
                for v in range(2):
                    a = util.view_args(scs[s], view=v)
                    ad = _depth_oracle_args(a, scs[s], mode, v)
                    f = util.oracle_forward(ad, (0, 0, 0), 64, 64)
                    _image_bar(depth[s, v].cpu().numpy(), f.color[0])
                    _image_bar(depth[s, v].cpu().numpy(), two[s, v].cpu().numpy())


def test_depth_forward_config1(cache):
    sc, bg = synthetic.scene_re10k_like(seed=0), (0.0, 0.0, 0.0)
    _check_depth_forward(cache, "config1", sc, bg, True, modes=("depth",))


@pytest.mark.parametrize("mode", MODES)
def test_depth_forward_matches_render_depth_views(mode):
    """render_views_with_depth against today's two-pass route on configs[0] and the re10k-like 64^2 scene."""
    from pixelsplat_b200.decoder.cuda_splatting import render_depth_views, render_views_with_depth
    for sc, bg in (_config0(), _re10k64()):
        t = lambda x: x.to(DEV)[None]
        cam = (t(sc.extrinsics[:1]), t(sc.intrinsics[:1]), t(sc.near[:1]), t(sc.far[:1]), sc.image_shape)
        with torch.no_grad():
            for si in (True, False):
                _, depth = render_views_with_depth(*cam, t(torch.tensor(bg))[:, None].float(), t(sc.means),
                                                   t(sc.covariances), t(sc.harmonics), t(sc.opacities), si, mode)
                two = render_depth_views(*cam, t(sc.means), t(sc.covariances), t(sc.opacities), si, mode)
                _image_bar(depth.cpu().numpy(), two.cpu().numpy())


# ------------------------------------------------------------------ 3. gradients against the oracle decomposition
def _oracle_depth_grads(cache, key, sc, bg, si, mode, d_img, d_dep):
    """(float32 reference, float64 reference) of the colour + depth gradients w.r.t. the native leaves."""
    a, n, s = _args(sc, bg, si)
    H, W = n["H"], n["W"]
    c32, c64 = _memo(cache, ("cgrad", key, si), lambda: util.oracle_gradients(a, bg, H, W, d_img))
    ad = _depth_oracle_args(a, sc, mode)
    dimg = np.stack([d_dep, np.zeros_like(d_dep), np.zeros_like(d_dep)]).astype(np.float32)
    d32, d64 = util.oracle_gradients(ad, (0, 0, 0), H, W, dimg)
    ch = _chain(sc, mode)
    # the depth-as-colour oracle's dL/dcolours[:, 0] is dL/dd, chained to the means in float64
    return [dict(means=s * (c["means"] + d["means"]) + np.asarray(d["col"], np.float64)[:, :1] * ch,
                 cov=s * s * (c["cov"] + d["cov"]), opac=c["opac"] + d["opac"], col=c["col"])
            for c, d in ((c32, d32), (c64, d64))]


def _check_depth_grads(got, ref32, ref64, tag):
    rep = {}
    for k in ("means", "cov", "opac", "col"):
        g = got[k].detach().cpu().numpy()
        r32 = util.grad_errors(g, ref32[k])
        rep[k] = r32
        assert r32["max"] <= 2e-3 and r32["l2"] <= util.L2_BAR and r32["q999"] <= 1.0, (tag, k, r32)
        r64, own = util.grad_errors(g, ref64[k]), util.grad_errors(ref32[k], ref64[k])
        assert r64["l2"] <= max(1.5 * own["l2"], 1e-5), (tag, k, r64, own)
        assert r64["q999"] <= max(1.5 * own["q999"], 1.0), (tag, k, r64, own)
    print("DEPTH_GRAD", tag, {k: {m: f"{v:.1e}" for m, v in r.items()} for k, r in rep.items()})


@pytest.mark.parametrize("name", list(WARP_VARIANTS))
@pytest.mark.parametrize("mode", MODES)
def test_depth_gradients(cache, name, mode):
    sc, bg = _config0()
    _, n, _ = _args(sc, bg, True)
    H, W = n["H"], n["W"]
    rng = np.random.default_rng(7)
    d_img = rng.standard_normal((3, H, W)).astype(np.float32)
    d_dep = rng.standard_normal((H, W)).astype(np.float32)
    ref32, ref64 = _memo(cache, ("dgrad", mode), lambda: _oracle_depth_grads(cache, "config0", sc, bg, True, mode,
                                                                           d_img, d_dep))
    with util.composite_variant(*WARP_VARIANTS[name]):
        out = native(n, mode, d_img, d_dep)
    _check_depth_grads(out["grads"], ref32, ref64, (name, mode))


# ------------------------------------------------------------------ 4. the loss path
@pytest.mark.parametrize("mode", ["depth", "relative_disparity"])
def test_forward_mse_with_depth(mode):
    """forward_mse(depth_mode=...) returns forward's depth bit for bit; its gradients with a dL/dD added equal the
    unfused route (render -> torch sum of squares, same dL/dD) to 2e-5 norm-wise."""
    from pixelsplat_b200.decoder import DecoderSplattingCUDA, DecoderSplattingCUDACfg, Gaussians
    scs = [synthetic.scene_re10k_like(seed=30 + i, image_hw=(48, 80), target_views=3) for i in range(2)]
    t = lambda k: torch.stack([getattr(sc, k) for sc in scs]).to(DEV)
    dec = DecoderSplattingCUDA(DecoderSplattingCUDACfg("splatting_cuda"),
                               type("D", (), {"background_color": [0.1, 0.2, 0.3]})()).to(DEV)
    target = torch.rand(2, 3, 3, 48, 80, device=DEV, generator=torch.Generator(DEV).manual_seed(3))
    d_dep = torch.randn(2, 3, 48, 80, device=DEV, generator=torch.Generator(DEV).manual_seed(5))
    cam = (t("extrinsics"), t("intrinsics"), t("near"), t("far"), (48, 80))
    grads = []
    for fused in (True, False):
        leaves = [t(k).requires_grad_(True) for k in ("means", "covariances", "harmonics", "opacities")]
        g = Gaussians(*leaves)
        if fused:
            out, sse, _ = dec.forward_mse(g, *cam, target, depth_mode=mode)
            ref = dec.forward(g, *cam, depth_mode=mode)
            assert torch.equal(out.depth.detach(), ref.depth.detach())
            loss = sse.sum() + (out.depth * d_dep).sum()
        else:
            out = dec.forward(g, *cam, depth_mode=mode)
            loss = ((out.color - target) ** 2).sum() + (out.depth * d_dep).sum()
        loss.backward()
        grads.append([l.grad for l in leaves])
    for gf, gu in zip(*grads):
        e = float((gf - gu).norm() / gu.norm())
        assert e <= 2e-5, e


# ------------------------------------------------------------------ 5. end to end: a LossDepth step
def test_loss_depth_step_fused_against_two_pass():
    """LossDepth (re10k_depth_loss settings: sigma 12, second derivative) on the fused depth: dL/dD is taken once,
    then pushed through the fused pass and through today's two-pass route (render_views + render_depth_views)."""
    from pixelsplat_b200 import loss as L
    from pixelsplat_b200.decoder.cuda_splatting import render_depth_views, render_views, render_views_with_depth
    sc = synthetic.scene_re10k_like(seed=40, image_hw=(64, 64), target_views=2)
    t = lambda x: x.to(DEV)[None]
    cam = (t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far), (64, 64))
    bg = torch.zeros(1, 2, 3, device=DEV)
    image = torch.rand(1, 2, 3, 64, 64, device=DEV, generator=torch.Generator(DEV).manual_seed(8))
    ld = L.LossDepth(L.LossDepthCfgWrapper(L.LossDepthCfg(0.25, 12.0, True)))
    batch = {"target": {"near": cam[2], "far": cam[3], "image": image}}
    res = []
    for fused in (True, False):
        leaves = [t(x).requires_grad_(True) for x in (sc.means, sc.covariances, sc.harmonics, sc.opacities)]
        if fused:
            color, depth = render_views_with_depth(*cam, bg, *leaves)
        else:
            color = render_views(*cam, bg, *leaves)
            depth = render_depth_views(*cam, leaves[0], leaves[1], leaves[3])
        d = depth.detach().requires_grad_(True)
        value = ld(type("O", (), {"depth": d})(), batch)
        value.backward()
        if fused:
            d_dep = d.grad
        (depth * d_dep).sum().backward()
        res.append((float(value.detach()), [torch.zeros_like(l) if l.grad is None else l.grad for l in leaves]))
    (vf, gf), (vt, gt) = res
    assert abs(vf - vt) <= 1e-5 * abs(vt), (vf, vt)
    for k, (a, b) in enumerate(zip(gf, gt)):
        if b.abs().max() == 0:
            assert a.abs().max() == 0
            continue
        e = float((a - b).norm() / b.norm())
        assert e <= 1e-4, (k, e)


# ------------------------------------------------------------------ 6. graphs and the legacy compositor
def test_cuda_graph_replay_matches_eager():
    from pixelsplat_b200.decoder.cuda_splatting import render_views_with_depth
    sc = synthetic.scene_re10k_like(seed=50, image_hw=(64, 64), target_views=2)
    t = lambda x: x.to(DEV)[None]
    cam = (t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far), (64, 64))
    bg = torch.zeros(1, 2, 3, device=DEV)
    leaves = [t(x).requires_grad_(True) for x in (sc.means, sc.covariances, sc.harmonics, sc.opacities)]
    w_c = torch.randn(1, 2, 3, 64, 64, device=DEV)
    w_d = torch.randn(1, 2, 64, 64, device=DEV)

    def step():
        for l in leaves:
            l.grad = None
        color, depth = render_views_with_depth(*cam, bg, *leaves, mode="disparity")
        ((color * w_c).sum() + (depth * w_d).sum()).backward()
        return color.detach(), depth.detach(), [l.grad for l in leaves]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager = step()              # also sizes the binning capacity of this shape
        eager = [eager[0].clone(), eager[1].clone(), [g.clone() for g in eager[2]]]
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = step()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])
    for a, b in zip(out[2], eager[2]):
        assert float((a - b).abs().max()) <= 1e-6 * float(b.abs().max()) or torch.equal(a, b)


def test_legacy_compositor_has_no_depth_channel():
    """composite_impl = 1: the C forward refuses a depth descriptor before enqueuing anything, and the decoder falls
    back to today's two-pass result."""
    from pixelsplat_b200 import _lib
    from pixelsplat_b200.decoder import DecoderSplattingCUDA, DecoderSplattingCUDACfg, Gaussians
    from pixelsplat_b200.decoder.cuda_splatting import render_depth_views, render_views
    sc, bg = _config0()
    _, n, _ = _args(sc, bg, False)
    with util.composite_variant(1, 1, 0):
        desc = _lib.RasterDesc(1, 1, n["means"].shape[0], 25, 4, 0, 0, 64, 64, 0, 0, 100000, 0, 1)
        sz = _lib.sizes(desc)
        bufs = [torch.empty(b, dtype=torch.uint8, device=DEV) for b in (sz.geom_bytes, sz.binning_bytes,
                                                                         sz.image_bytes)]
        x = torch.zeros(1 << 16, device=DEV)
        inputs = _lib.RasterInputs(*([x.data_ptr()] * 9), None, None)
        state = _lib.RasterState(bufs[0].data_ptr(), sz.geom_bytes, bufs[1].data_ptr(), sz.binning_bytes,
                                 bufs[2].data_ptr(), sz.image_bytes)
        before = _lib.lib.ps_launch_count()
        rc = _lib.lib.ps_raster_forward(ctypes.byref(desc), ctypes.byref(inputs), ctypes.byref(state),
                                        ctypes.c_void_p(x.data_ptr()), None, None, None)
        assert rc == _lib.PS_ERR_UNSUPPORTED and b"legacy" in _lib.lib.ps_last_error()
        assert _lib.lib.ps_launch_count() == before
        dec = DecoderSplattingCUDA(DecoderSplattingCUDACfg("splatting_cuda"),
                                   type("D", (), {"background_color": [0.1, 0.2, 0.3]})()).to(DEV)
        t = lambda x: x.to(DEV)[None]
        cam = (t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far), sc.image_shape)
        g = Gaussians(t(sc.means), t(sc.covariances), t(sc.harmonics), t(sc.opacities))
        with torch.no_grad():
            out = dec(g, *cam, depth_mode="log")
            color = render_views(*cam, dec.background_color.expand(1, 1, 3), g.means, g.covariances, g.harmonics,
                                 g.opacities)
            depth = render_depth_views(*cam, g.means, g.covariances, g.opacities, mode="log")
        assert torch.equal(out.color, color) and torch.equal(out.depth, depth)
