"""GPU tests of SSIM (csrc/ssim.cu through pixelsplat_b200.loss.ssim / compute_ssim) against the float64
restatements of the reference's compute_ssim (/root/reference/src/evaluation/metrics.py:36-52) in
oracle/ssim_oracle.py: the forward per plane to 1e-5 absolute, the backward against torch float64 autograd of the
oracle to 1e-4 norm-wise, exact properties (ssim(x, x) = 1, symmetry, determinism, graph replay) and the chain into
the rasterizer's backward.  Worst errors are printed (run with -s to see them)."""
import numpy as np
import pytest
import torch

from oracle import ssim_oracle as so
from pixelsplat_b200 import synthetic

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FWD_BAR = 1e-5
BWD_BAR = 1e-4


def _render(sc, bg=(0.0, 0.0, 0.0)) -> torch.Tensor:
    """[V, 3, h, w] render of a synthetic scene (no gradient)."""
    from pixelsplat_b200.decoder import render_views
    t = lambda x: x.to(DEV)[None]
    V = sc.extrinsics.shape[0]
    with torch.no_grad():
        img = render_views(t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far), sc.image_shape,
                           torch.tensor(bg, device=DEV).expand(1, V, 3), t(sc.means), t(sc.covariances),
                           t(sc.harmonics), t(sc.opacities))
    return img[0].contiguous()


def _input(kind: str):
    """(ground truth, prediction) [b, c, h, w] float32 on the device."""
    g = torch.Generator().manual_seed(17 + KINDS.index(kind))
    r = lambda *s: torch.rand(s, generator=g)
    if kind == "noise":
        x, y = r(3, 3, 64, 80), r(3, 3, 64, 80)
    elif kind == "smooth":
        yy, xx = torch.meshgrid(torch.arange(96) / 30.0, torch.arange(72) / 30.0, indexing="ij")
        base = torch.stack([0.5 + 0.3 * torch.sin(3 * xx + k) * torch.cos(2 * yy - k) for k in range(3)])[None]
        x = base + 0.01 * torch.randn((2, 3, 96, 72), generator=g)
        y = base + 0.01 * torch.randn((2, 3, 96, 72), generator=g)
    elif kind == "flat_bright":
        x, y = 0.95 + 0.002 * (2 * r(2, 3, 64, 64) - 1), 0.95 + 0.002 * (2 * r(2, 3, 64, 64) - 1)
    elif kind == "above_one":
        x, y = 1.6 * r(2, 3, 40, 50), 0.3 + 1.4 * r(2, 3, 40, 50)
    elif kind in ("render_config0", "render_re10k256"):
        sc = (synthetic.scene_random_frustum(seed=0) if kind == "render_config0"
              else synthetic.scene_re10k_like(seed=3, image_hw=(256, 256), target_views=2))
        x = _render(sc).cpu()
        y = x + 0.03 * torch.randn(x.shape, generator=g)
    else:
        raise KeyError(kind)
    return x.float().to(DEV).contiguous(), y.float().to(DEV).contiguous()


KINDS = ["noise", "smooth", "flat_bright", "above_one", "render_config0", "render_re10k256"]
SHAPES = [(1, 1, 11, 11), (1, 1, 11, 300), (1, 1, 300, 11), (2, 3, 257, 255), (1, 3, 512, 512), (1, 1, 64, 64),
          (32, 3, 40, 33), (32, 3, 256, 256)]


def _planes(t: torch.Tensor) -> torch.Tensor:
    """[b, c, h, w] -> [b c, 1, h, w]: ssim of these gives one score per plane."""
    b, c, h, w = t.shape
    return t.reshape(b * c, 1, h, w)


def _check_forward(x, y, tag):
    from pixelsplat_b200.loss import ssim
    got = ssim(_planes(x), _planes(y)).double().cpu().numpy()
    ref = so.ssim_planes_torch(x.double(), y.double()).reshape(-1).cpu().numpy()
    err = np.abs(got - ref).max()
    print(f"[ssim fwd] {tag}: planes {ref.size}, max |err| {err:.2e}, score range [{ref.min():.4f}, {ref.max():.4f}]")
    assert err <= FWD_BAR, (tag, err)
    # the image score is the channel mean
    img = ssim(x, y).double().cpu().numpy()
    assert np.abs(img - ref.reshape(x.shape[:2]).mean(axis=1)).max() <= FWD_BAR
    return err


def _check_backward(x, y, tag):
    from pixelsplat_b200.loss import ssim
    n = x.shape[0] * x.shape[1]
    w = torch.randn(n, generator=torch.Generator().manual_seed(n)).to(DEV)
    xg, yg = _planes(x).clone().requires_grad_(True), _planes(y).clone().requires_grad_(True)
    (ssim(xg, yg) * w).sum().backward()
    x64, y64 = x.double().requires_grad_(True), y.double().requires_grad_(True)
    (so.ssim_planes_torch(x64, y64).reshape(-1) * w.double()).sum().backward()
    out = {}
    for name, got, ref in (("dy", yg.grad, y64.grad), ("dx", xg.grad, x64.grad)):
        got, ref = got.reshape(ref.shape).double(), ref
        rel = float((got - ref).norm() / ref.norm())
        mx = float((got - ref).abs().max())
        out[name] = rel
        print(f"[ssim bwd] {tag} {name}: |got - ref| / |ref| {rel:.2e}, max |err| {mx:.2e}, max |ref| "
              f"{float(ref.abs().max()):.2e}")
        assert rel <= BWD_BAR, (tag, name, rel)
        # the 5-pixel frame outside the crop has gradient (its pixels lie in the windows of crop pixels)
        frame = torch.ones(ref.shape[-2:], dtype=torch.bool, device=DEV)
        frame[5:-5, 5:-5] = False
        gf, rf = got[..., frame], ref[..., frame]
        assert float(rf.abs().max()) > 0 and float(gf.abs().max()) > 0
        assert float((gf - rf).norm()) <= BWD_BAR * float(rf.norm()) + 1e-12, (tag, name, "frame")
    return out


@pytest.mark.parametrize("kind", KINDS)
def test_forward_matches_the_float64_oracle(kind):
    x, y = _input(kind)
    _check_forward(x, y, kind)
    # the numpy restatement (filter written out, reflect padding) on one plane agrees as well
    ref_np = so.ssim_plane_numpy(x[0, 0].double().cpu().numpy(), y[0, 0].double().cpu().numpy())
    from pixelsplat_b200.loss import ssim
    got = float(ssim(x[:1, :1], y[:1, :1]))
    assert abs(got - ref_np) <= FWD_BAR


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_forward_shapes(shape):
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.rand(shape, generator=g).to(DEV)
    y = (x.cpu() + 0.2 * torch.randn(shape, generator=g)).to(DEV)
    _check_forward(x, y, "shape " + "x".join(map(str, shape)))


@pytest.mark.parametrize("kind", KINDS)
def test_backward_matches_float64_autograd(kind):
    x, y = _input(kind)
    _check_backward(x, y, kind)


@pytest.mark.parametrize("shape", [(1, 1, 11, 11), (1, 1, 11, 300), (1, 1, 300, 11), (2, 3, 257, 255),
                                   (1, 3, 512, 512), (32, 3, 256, 256)], ids=lambda s: "x".join(map(str, s)))
def test_backward_shapes(shape):
    g = torch.Generator().manual_seed(sum(shape) + 1)
    x = torch.rand(shape, generator=g).to(DEV)
    y = (x.cpu() + 0.2 * torch.randn(shape, generator=g)).to(DEV)
    _check_backward(x, y, "shape " + "x".join(map(str, shape)))


def test_ground_truth_gradient_only_when_required():
    from pixelsplat_b200.loss import ssim
    x, y = _input("noise")
    yg = y.clone().requires_grad_(True)
    ssim(x, yg).sum().backward()
    assert x.grad is None and yg.grad is not None and bool(torch.isfinite(yg.grad).all())
    y64 = y.double().requires_grad_(True)
    so.ssim_torch(x.double(), y64).sum().backward()
    assert float((yg.grad.double() - y64.grad).norm() / y64.grad.norm()) <= BWD_BAR


def test_exact_properties():
    from pixelsplat_b200.loss import ssim
    for kind in ("noise", "flat_bright", "render_config0"):
        x, y = _input(kind)
        one = ssim(x, x)
        assert float((one - 1).abs().max()) <= 1e-6, kind
        a, b = ssim(x, y), ssim(y, x)
        assert float((a - b).abs().max()) <= 1e-7, kind
        assert torch.equal(ssim(x, y), a), kind                       # the same bits every call
    # non-contiguous inputs are made contiguous
    x, y = _input("noise")
    xt, yt = x.transpose(-1, -2).contiguous().transpose(-1, -2), y.transpose(-1, -2).contiguous().transpose(-1, -2)
    assert not xt.is_contiguous() and torch.equal(ssim(xt, yt), ssim(x, y))


def test_cuda_graph_replay_equals_eager():
    from pixelsplat_b200.loss import ssim
    x, y = _input("smooth")
    xs, ys = x.clone(), y.clone()
    yg = ys.clone().requires_grad_(True)
    eager = ssim(x, y)
    eager_grad = torch.autograd.grad(ssim(x, yg).sum(), yg)[0]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                        # warm-up outside the capture
        ssim(xs, ys)
        torch.autograd.grad(ssim(xs, yg).sum(), yg)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ssim(xs, ys)
        gout = torch.autograd.grad(ssim(xs, yg).sum(), yg)[0]
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager) and torch.equal(gout, eager_grad)
    # new inputs in the captured buffers give the new answer
    x2 = torch.rand(x.shape, generator=torch.Generator().manual_seed(9)).to(DEV)
    xs.copy_(x2)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, ssim(x2, y))


def test_end_to_end_into_the_rasterizer():
    """(1 - ssim(target, render)).mean() backpropagated into the Gaussians equals the rasterizer's backward fed with
    the oracle's float64 dL/dC."""
    from pixelsplat_b200.decoder import render_views
    from pixelsplat_b200.loss import ssim
    sc = synthetic.scene_re10k_like(seed=12, image_hw=(128, 128), target_views=2)
    t = lambda x: x.to(DEV)[None]
    cam = (t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far), sc.image_shape)
    bg = torch.zeros(1, 2, 3, device=DEV)
    target = (_render(sc).cpu() + 0.05 * torch.randn((2, 3, 128, 128), generator=torch.Generator().manual_seed(4))
              ).to(DEV)

    def leaves():
        return [t(getattr(sc, k)).requires_grad_(True) for k in ("means", "covariances", "harmonics", "opacities")]

    la = leaves()
    img = render_views(*cam, bg, *la)[0]
    (1 - ssim(target, img)).mean().backward()
    lb = leaves()
    img_b = render_views(*cam, bg, *lb)[0]
    c64 = img_b.detach().double().requires_grad_(True)
    (1 - so.ssim_torch(target.double(), c64)).mean().backward()
    img_b.backward(c64.grad.float())
    for name, a, b in zip(("means", "covariances", "harmonics", "opacities"), la, lb):
        rel = float((a.grad - b.grad).norm() / b.grad.norm())
        print(f"[ssim e2e] d{name}: |got - ref| / |ref| {rel:.2e}")
        assert float(b.grad.norm()) > 0 and rel <= BWD_BAR, (name, rel)


def test_compute_ssim_is_the_metric():
    from pixelsplat_b200.loss import compute_ssim, ssim
    x, y = _input("render_config0")
    yg = y.clone().requires_grad_(True)
    got = compute_ssim(x, yg)
    assert got.shape == (x.shape[0],) and got.dtype == torch.float32 and got.device == y.device
    assert not got.requires_grad and torch.equal(got, ssim(x, y))
    ref = so.ssim_numpy(x.double().cpu().numpy(), y.double().cpu().numpy())
    assert np.abs(got.double().cpu().numpy() - ref).max() <= FWD_BAR
