"""GPU tests of the fused loss epilogue (SURVEY.md 8 row f-4): the compositor's per-view squared-error sums and
the in-kernel dL/dC against the unfused route -- render, then the reference's LossMse
(/root/reference/src/loss/loss_mse.py:30-31) and compute_psnr (src/evaluation/metrics.py:11-19) in torch."""
import pytest
import torch

from pixelsplat_b200 import synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _decoder():
    from pixelsplat_b200.decoder import DecoderSplattingCUDA, DecoderSplattingCUDACfg
    return DecoderSplattingCUDA(DecoderSplattingCUDACfg("splatting_cuda"),
                                type("D", (), {"background_color": [0.1, 0.0, 0.2]})()).to(DEV)


# the warp-task compositor variants: (composite_impl, composite_segments, composite_hit_lists)
VARIANTS = {"k1": (2, 1, 1), "k1-nohl": (2, 1, 0), "k2": (2, 2, 1), "k2-nohl": (2, 2, 0), "k4": (2, 4, 1),
            "k4-nohl": (2, 4, 0)}


@pytest.mark.parametrize("hw,views", [((64, 64), 1), ((48, 80), 3), ((256, 256), 4)])
def test_fused_mse_and_psnr_equal_the_unfused_route(hw, views):
    """The compositor variant the shape selects automatically."""
    _fused_equals_unfused(hw, views)


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_fused_mse_and_psnr_equal_the_unfused_route_under_every_variant(variant):
    """The (48, 80) x 3 case with each warp-task variant forced; both routes run under the same variant."""
    from tests import util
    with util.composite_variant(*VARIANTS[variant]):
        _fused_equals_unfused((48, 80), 3)


def _fused_equals_unfused(hw, views):
    from pixelsplat_b200 import loss as L
    from pixelsplat_b200.decoder import Gaussians
    S = 2
    scs = [synthetic.scene_re10k_like(seed=70 + i, image_hw=(32, 32) if hw[0] < 256 else hw, target_views=views)
           for i in range(S)]
    st = lambda name: torch.stack([getattr(s, name).to(DEV) for s in scs])
    dec = _decoder()
    g = torch.Generator().manual_seed(3)
    target = (torch.rand((S, views, 3, *hw), generator=g) * 1.4 - 0.2).to(DEV)      # some values outside [0, 1]
    weight = 0.7

    def leaves():
        return Gaussians(st("means").requires_grad_(True), st("covariances").requires_grad_(True),
                         st("harmonics").requires_grad_(True), st("opacities").requires_grad_(True))

    cams = (st("extrinsics"), st("intrinsics"), st("near"), st("far"), hw)
    # unfused: render, LossMse, compute_psnr
    ga = leaves()
    out = dec(ga, *cams)
    mse = L.LossMse(L.LossMseCfgWrapper(L.LossMseCfg(weight)))
    loss_a = mse(out, {"target": {"image": target}})
    loss_a.backward()
    psnr_a = L.compute_psnr(target.flatten(0, 1), out.color.detach().flatten(0, 1)).reshape(S, views)
    # fused
    gb = leaves()
    out_b, sse, sse_clipped = dec.forward_mse(gb, *cams, target)
    loss_b = mse.from_sse(sse, hw)
    loss_b.backward()
    psnr_b = L.psnr_from_sse(sse_clipped, hw)
    assert torch.equal(out_b.color, out.color.detach())                              # same compositor, same pixels
    assert abs(float(loss_a) - float(loss_b)) <= 2e-6 * abs(float(loss_a))
    assert torch.allclose(psnr_a, psnr_b, atol=1e-4)
    for name in ("means", "covariances", "harmonics", "opacities"):
        a, b = getattr(ga, name).grad, getattr(gb, name).grad
        assert (a - b).norm() <= 2e-5 * a.norm(), name                              # atomics order only
    # want_color=False: no image tensor at all, same numbers
    gc = leaves()
    out_c, sse_c, _ = dec.forward_mse(gc, *cams, target, want_color=False)
    assert out_c.color is None and torch.allclose(sse_c, sse.detach(), rtol=1e-6)
    # a per-view weighting of the sums reaches the kernel as a per-view gradient scale
    gd = leaves()
    wv = torch.linspace(0.5, 2.0, S * views, device=DEV).reshape(S, views)
    _, sse_d, _ = dec.forward_mse(gd, *cams, target)
    (sse_d * wv).sum().backward()
    ge = leaves()
    out_e = dec(ge, *cams)
    (((out_e.color - target) ** 2).sum(dim=(2, 3, 4)) * wv).sum().backward()
    assert (gd.means.grad - ge.means.grad).norm() <= 2e-5 * ge.means.grad.norm()
    assert (gd.harmonics.grad - ge.harmonics.grad).norm() <= 2e-5 * ge.harmonics.grad.norm()


def test_fused_gradients_agree_across_list_runs():
    """The fused loss's gradients with K = 2 list runs per task against K = 1 (one warp walks the whole list)."""
    from pixelsplat_b200.decoder import Gaussians
    from tests import util
    S, views, hw = 2, 3, (48, 80)
    scs = [synthetic.scene_re10k_like(seed=70 + i, image_hw=(32, 32), target_views=views) for i in range(S)]
    st = lambda name: torch.stack([getattr(s, name).to(DEV) for s in scs])
    cams = (st("extrinsics"), st("intrinsics"), st("near"), st("far"), hw)
    target = (torch.rand((S, views, 3, *hw), generator=torch.Generator().manual_seed(3)) * 1.4 - 0.2).to(DEV)
    dec = _decoder()
    grads = {}
    for K in (1, 2):
        g = Gaussians(st("means").requires_grad_(True), st("covariances").requires_grad_(True),
                      st("harmonics").requires_grad_(True), st("opacities").requires_grad_(True))
        with util.composite_variant(2, K, 2):
            _, sse, _ = dec.forward_mse(g, *cams, target)
            sse.sum().backward()
        grads[K] = {n: getattr(g, n).grad for n in ("means", "covariances", "harmonics", "opacities")}
    for n, a in grads[1].items():
        assert (grads[2][n] - a).norm() <= 1e-4 * a.norm(), n


def test_legacy_compositor_rejects_the_loss_epilogue():
    from pixelsplat_b200 import _lib
    from pixelsplat_b200.decoder import Gaussians
    sc = synthetic.scene_random_frustum(seed=1)
    dec = _decoder()
    g = Gaussians(*[t.to(DEV)[None] for t in (sc.means, sc.covariances, sc.harmonics, sc.opacities)])
    cams = tuple(t.to(DEV)[None] for t in (sc.extrinsics, sc.intrinsics, sc.near, sc.far)) + (sc.image_shape,)
    _lib.set_option("composite_impl", 1)
    try:
        with pytest.raises(_lib.NativeError, match="legacy compositor"):
            dec.forward_mse(g, *cams, torch.zeros(1, 1, 3, *sc.image_shape, device=DEV))
    finally:
        _lib.set_option("composite_impl", 2)
