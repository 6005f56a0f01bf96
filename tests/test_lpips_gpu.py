"""GPU tests of LPIPS (csrc/lpips.cu through pixelsplat_b200.lpips and the LossLpips / compute_lpips drop-ins) against
the float64 restatement of the lpips package's LPIPS(net="vgg") in oracle/lpips_oracle.py: the fused head forward per
image to 1e-5 relative and backward per layer to 2e-5 norm-wise on the same float32 features, exact cases, train-mode
dropout against the numpy restatement of the hash, the whole module with random weights, determinism, graph replay
and the chain into the rasterizer's backward.  Worst errors are printed (run with -s to see them)."""
import numpy as np
import pytest
import torch

from oracle import lpips_oracle as lo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FWD_BAR = 1e-5
BWD_BAR = 2e-5
WHOLE_BAR = 1e-4          # whole module, TF32 off
# its input gradient, TF32 off: float32 and float64 trunks route a few ReLU / max-pool gradients differently
WHOLE_GRAD_BAR = 1e-3
WHOLE_BAR_TF32 = 1e-3     # whole module under torch's default cuDNN settings (TF32 convolutions)


def _vgg_shapes(h, w, n_layers=5):
    shapes = []
    for c in lo.CHANNELS[:n_layers]:
        shapes.append((c, h, w))
        h, w = h // 2, w // 2
    return shapes


def _features(N, shapes, seed, near=False):
    """ReLU-sparse float32 feature pairs on the device (`near`: x1 a small perturbation of x0)."""
    g = torch.Generator().manual_seed(seed)
    f0 = [torch.relu(torch.randn((N, *s), generator=g)) for s in shapes]
    if near:
        f1 = [torch.relu(a + 1e-3 * torch.randn(a.shape, generator=g)) for a in f0]
    else:
        f1 = [torch.relu(torch.randn((N, *s), generator=g)) for s in shapes]
    w = [torch.rand(s[0], generator=g) for s in shapes]
    return [t.to(DEV) for t in f0], [t.to(DEV) for t in f1], [t.to(DEV) for t in w]


CASES = {
    "vgg256_n3": (3, _vgg_shapes(256, 256)),
    "odd255x257_n1": (1, _vgg_shapes(255, 257)),
    "in16x16_n28": (28, _vgg_shapes(16, 16)),
    "vgg64_n3_1layer": (3, _vgg_shapes(64, 64, 1)),
    "vgg64_n3_2layers": (3, _vgg_shapes(64, 64, 2)),
    "vgg64_n3_3layers": (3, _vgg_shapes(64, 64, 3)),
    "vgg64_n3_4layers": (3, _vgg_shapes(64, 64, 4)),
    "vgg64_n28_5layers": (28, _vgg_shapes(64, 64)),
    "odd_channels": (2, [(3, 17, 9), (200, 5, 31), (8192, 1, 3)]),
}


def _masks(seed, f0):
    return [torch.from_numpy(lo.dropout_mask(seed, l, tuple(t.shape))) for l, t in enumerate(f0)]


def _check_forward(f0, f1, w, tag, seed=None):
    from pixelsplat_b200.lpips import lpips_head
    st = None if seed is None else torch.tensor([seed], dtype=torch.int64, device=DEV)
    got = lpips_head(f0, f1, w, st).double().cpu()
    masks = None if seed is None else _masks(seed, f0)
    ref = lo.head([t.double().cpu() for t in f0], [t.double().cpu() for t in f1], [t.double().cpu() for t in w], masks)
    rel = float(((got - ref).abs() / ref.abs()).max())
    print(f"[lpips head fwd] {tag}: N {ref.numel()}, max rel err {rel:.2e}, value range [{float(ref.min()):.4g}, "
          f"{float(ref.max()):.4g}]")
    assert got.shape == ref.shape and rel <= FWD_BAR, (tag, rel)
    return rel


def _check_backward(f0, f1, w, tag, sides=(0, 1), seed=None):
    from pixelsplat_b200.lpips import lpips_head
    N = f0[0].shape[0]
    dout = torch.randn(N, generator=torch.Generator().manual_seed(N + 1)).to(DEV)
    a = [t.clone().requires_grad_(0 in sides) for t in f0]
    b = [t.clone().requires_grad_(1 in sides) for t in f1]
    st = None if seed is None else torch.tensor([seed], dtype=torch.int64, device=DEV)
    (lpips_head(a, b, w, st) * dout).sum().backward()
    a64 = [t.double().cpu().requires_grad_(True) for t in f0]
    b64 = [t.double().cpu().requires_grad_(True) for t in f1]
    masks = None if seed is None else _masks(seed, f0)
    (lo.head(a64, b64, [t.double().cpu() for t in w], masks) * dout.double().cpu()).sum().backward()
    worst = 0.0
    for side, got, ref in ((0, a, a64), (1, b, b64)):
        for l, (g, r) in enumerate(zip(got, ref)):
            if side not in sides:
                assert g.grad is None
                continue
            # float64 autograd is NaN at an all-zero column (sqrt's derivative at 0; test_exact_cases checks the
            # kernel's limit there), which ReLU-sparse maps with few channels have
            ok = torch.isfinite(r.grad)
            rel = float((g.grad.double().cpu()[ok] - r.grad[ok]).norm() / r.grad[ok].norm())
            worst = max(worst, rel)
            assert rel <= BWD_BAR, (tag, side, l, rel)
    print(f"[lpips head bwd] {tag} sides {sides}: worst per-layer norm-wise rel err {worst:.2e}")
    return worst


@pytest.mark.parametrize("case", list(CASES))
def test_head_forward_matches_float64(case):
    N, shapes = CASES[case]
    f0, f1, w = _features(N, shapes, seed=len(case))
    _check_forward(f0, f1, w, case)
    f0, f1, w = _features(N, shapes, seed=len(case) + 50, near=True)
    _check_forward(f0, f1, w, case + " near")


@pytest.mark.parametrize("case", ["vgg256_n3", "odd255x257_n1", "in16x16_n28", "vgg64_n3_2layers", "odd_channels"])
@pytest.mark.parametrize("sides", [(0, 1), (0,), (1,)], ids=["both", "x0", "x1"])
def test_head_backward_matches_float64_autograd(case, sides):
    N, shapes = CASES[case]
    f0, f1, w = _features(N, shapes, seed=len(case) + 7)
    _check_backward(f0, f1, w, case, sides)


def test_exact_cases():
    from pixelsplat_b200.lpips import lpips_head
    f0, f1, w = _features(3, _vgg_shapes(64, 64), seed=3)
    a = [t.clone().requires_grad_(True) for t in f0]
    b = [t.clone().requires_grad_(True) for t in f0]
    out = lpips_head(a, b, w)
    assert float(out.detach().abs().max()) == 0.0
    out.sum().backward()
    assert all(float(t.grad.abs().max()) == 0.0 for t in a + b)
    # an all-zero column of x0 at one pixel: the analytic limit z / eps there (autograd of the formula is NaN)
    f0, f1, w = _features(2, [(64, 8, 8)], seed=4)
    f0[0][1, :, 3, 5] = 0.0
    a = [f0[0].clone().requires_grad_(True)]
    b = [f1[0].clone().requires_grad_(True)]
    dout = torch.tensor([0.7, -1.3], device=DEV)
    (lpips_head(a, b, w) * dout).sum().backward()
    x1 = f1[0][1, :, 3, 5].double()
    u = -x1 / (x1.norm() + 1e-10)
    z = 2 * w[0].double() * float(dout[1]) / 64 * u
    got = a[0].grad[1, :, 3, 5].double()
    rel = float((got - z / 1e-10).norm() / (z / 1e-10).norm())
    print(f"[lpips zero column] limit z/eps: rel err {rel:.2e}, |d x0| {float(got.norm()):.3e}")
    assert rel <= 1e-5 and bool(torch.isfinite(a[0].grad).all() and torch.isfinite(b[0].grad).all())
    # everywhere else the gradient matches float64 autograd
    a64, b64 = f0[0].double().cpu().requires_grad_(True), f1[0].double().cpu().requires_grad_(True)
    (lo.head([a64], [b64], [w[0].double().cpu()]) * dout.double().cpu()).sum().backward()
    keep = torch.ones_like(a64, dtype=torch.bool)
    keep[1, :, 3, 5] = False
    ga = a[0].grad.double().cpu()
    assert float((ga[keep] - a64.grad[keep]).norm() / a64.grad[keep].norm()) <= BWD_BAR
    assert float((b[0].grad.double().cpu() - b64.grad).norm() / b64.grad.norm()) <= BWD_BAR


def test_train_mode_dropout_matches_the_hash():
    from pixelsplat_b200.lpips import lpips_head
    for case in ("vgg64_n28_5layers", "odd255x257_n1"):
        N, shapes = CASES[case]
        f0, f1, w = _features(N, shapes, seed=11)
        for seed in (0, -7, 2 ** 62 + 12345):
            _check_forward(f0, f1, w, f"{case} dropout seed {seed}", seed=seed)
        _check_backward(f0, f1, w, f"{case} dropout", (0, 1), seed=123456789)
        _check_backward(f0, f1, w, f"{case} dropout", (0,), seed=-5)
    f0, f1, w = _features(3, _vgg_shapes(64, 64), seed=12)
    s = lambda v: torch.tensor([v], dtype=torch.int64, device=DEV)
    a, b, ev = lpips_head(f0, f1, w, s(1)), lpips_head(f0, f1, w, s(2)), lpips_head(f0, f1, w)
    assert not torch.equal(a, b) and torch.equal(a, lpips_head(f0, f1, w, s(1)))
    # E[m] = 1: the dropout value scatters around the eval value
    vals = torch.stack([lpips_head(f0, f1, w, s(k)) for k in range(32)])
    assert float(((vals.mean(0) - ev).abs() / ev).max()) < 0.02


def _module(seed=0):
    from pixelsplat_b200.lpips import Lpips
    m = Lpips()
    m.load_state_dict(lo.random_state_dict(seed))
    return m.to(DEV).eval()


def _images(N, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand((N, 3, h, w), generator=g)
    b = (a + 0.1 * torch.randn(a.shape, generator=g)).clamp(0, 1)
    return a.to(DEV), b.to(DEV)


@pytest.mark.parametrize("shape", [(2, 64, 64), (1, 255, 257), (4, 16, 16)], ids=lambda s: "x".join(map(str, s)))
def test_whole_module_matches_float64(shape):
    m = _module(1)
    sd = {k: v.double() for k, v in lo.random_state_dict(1).items()}
    a, b = _images(*shape, seed=sum(shape))
    ref = lo.lpips(a.double().cpu(), b.double().cpu(), sd, normalize=True).reshape(-1)
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    try:
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        got = m(a, b, normalize=True)
        assert got.shape == (shape[0], 1, 1, 1)
        rel = float(((got.reshape(-1).double().cpu() - ref).abs() / ref).max())
        # the gradient through the trunk (target without grad)
        ag = a.clone().requires_grad_(True)
        m(ag, b, normalize=True).sum().backward()
        a64 = a.double().cpu().requires_grad_(True)
        lo.lpips(a64, b.double().cpu(), sd, normalize=True).sum().backward()
        grel = float((ag.grad.double().cpu() - a64.grad).norm() / a64.grad.norm())
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    got32 = m(a, b, normalize=True)
    rel32 = float(((got32.reshape(-1).double().cpu() - ref).abs() / ref).max())
    print(f"[lpips whole] {shape}: TF32 off max rel {rel:.2e}, grad norm-wise {grel:.2e}; cuDNN default "
          f"(allow_tf32={torch.backends.cudnn.allow_tf32}) max rel {rel32:.2e}")
    assert rel <= WHOLE_BAR and grel <= WHOLE_GRAD_BAR and rel32 <= WHOLE_BAR_TF32


def test_determinism():
    """Repeated forward + backward calls of the head give identical bits, with and without the deterministic flag."""
    from pixelsplat_b200.lpips import lpips_head
    f0, f1, w = _features(3, _vgg_shapes(64, 64), seed=6)

    def run(seed):
        x = [t.clone().requires_grad_(True) for t in f0]
        y = [t.clone().requires_grad_(True) for t in f1]
        o = lpips_head(x, y, w, None if seed is None else torch.tensor([seed], dtype=torch.int64, device=DEV))
        (o * torch.arange(1.0, 4.0, device=DEV)).sum().backward()
        return [o.detach()] + [t.grad for t in x + y]

    for seed in (None, 3):
        runs = [run(seed) for _ in range(3)]
        torch.use_deterministic_algorithms(True)
        try:
            runs.append(run(seed))
        finally:
            torch.use_deterministic_algorithms(False)
        for r in runs[1:]:
            assert all(torch.equal(p, q) for p, q in zip(runs[0], r)), seed


def _loss(weight=0.05, after=0, seed=3):
    from pixelsplat_b200.loss import LossLpips, LossLpipsCfg, LossLpipsCfgWrapper
    return LossLpips(LossLpipsCfgWrapper(LossLpipsCfg(weight, after)), lpips=_module(seed)).to(DEV)


def test_cuda_graph_replay_of_the_loss():
    loss = _loss().eval()
    g = torch.Generator().manual_seed(8)
    pred = torch.rand((1, 2, 3, 64, 64), generator=g).to(DEV).requires_grad_(True)
    batch = {"target": {"image": torch.rand((1, 2, 3, 64, 64), generator=g).to(DEV)}}
    P = type("P", (), {})

    def step():
        p = P()
        p.color = pred
        val = loss(p, batch, None, 10)
        return val.detach(), torch.autograd.grad(val, pred)[0]

    eager_val, eager_grad = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gval, ggrad = step()
    graph.replay()
    torch.cuda.synchronize()
    print(f"[lpips graph] eager {float(eager_val):.6f} replay {float(gval):.6f}")
    assert torch.allclose(gval, eager_val, rtol=1e-6, atol=0) and torch.allclose(ggrad, eager_grad, rtol=1e-5,
                                                                                 atol=1e-9)
    eager2 = step()
    assert torch.equal(eager2[0], eager_val) or float((eager2[0] - eager_val).abs()) <= 1e-6 * float(eager_val)


def test_train_mode_module_draws_a_new_mask_each_forward():
    loss = _loss()
    a, b = _images(2, 32, 32, seed=9)
    m = loss.lpips
    m.train()
    v1, v2 = m(a, b, normalize=True), m(a, b, normalize=True)
    m.eval()
    e1, e2 = m(a, b, normalize=True), m(a, b, normalize=True)
    assert not torch.equal(v1, v2) and torch.equal(e1, e2)


@pytest.fixture
def deterministic_fp32():
    """Fixed-order rasterizer and cuDNN gradients and no TF32, so that the two chains differ only in the head."""
    old = (torch.backends.cudnn.allow_tf32, torch.are_deterministic_algorithms_enabled())
    torch.backends.cudnn.allow_tf32 = False
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.backends.cudnn.allow_tf32 = old[0]
    torch.use_deterministic_algorithms(old[1])


def test_end_to_end_into_the_rasterizer(deterministic_fp32):
    """MSE + LossLpips of render_views backpropagated into the Gaussians equals the same chain with the torch head
    (the oracle's form in float32 on the same trunk)."""
    from pixelsplat_b200 import synthetic
    from pixelsplat_b200.decoder import render_views
    sc = synthetic.scene_re10k_like(seed=12, image_hw=(128, 128), target_views=2)
    t = lambda x: x.to(DEV)[None]
    cam = (t(sc.extrinsics), t(sc.intrinsics), t(sc.near), t(sc.far), sc.image_shape)
    bg = torch.zeros(1, 2, 3, device=DEV)
    loss = _loss(0.05, 150_000).eval()
    m = loss.lpips
    with torch.no_grad():
        target = (render_views(*cam, bg, *[t(getattr(sc, k)) for k in ("means", "covariances", "harmonics",
                                                                      "opacities")])
                  + 0.05 * torch.randn((1, 2, 3, 128, 128), generator=torch.Generator().manual_seed(4)).to(DEV))
    batch = {"target": {"image": target.clamp(0, 1)}}

    def leaves():
        return [t(getattr(sc, k)).requires_grad_(True) for k in ("means", "covariances", "harmonics", "opacities")]

    P = type("P", (), {})
    la = leaves()
    p = P()
    p.color = render_views(*cam, bg, *la)
    assert float(loss(p, batch, None, 149_999)) == 0.0                     # gated off before apply_after_step
    total = (p.color - batch["target"]["image"]).square().mean() + loss(p, batch, None, 150_000)
    total.backward()

    lb = leaves()
    img = render_views(*cam, bg, *lb)
    x0 = m.features(img.flatten(0, 1), True)
    with torch.no_grad():
        x1 = m.features(batch["target"]["image"].flatten(0, 1), True)
    torch_head = lo.head(x0, x1, m.lin_weights())
    total_b = (img - batch["target"]["image"]).square().mean() + 0.05 * torch_head.mean()
    total_b.backward()
    print(f"[lpips e2e] loss fused {float(total):.7f} torch head {float(total_b):.7f}")
    assert abs(float(total) - float(total_b)) <= 1e-5 * abs(float(total_b))
    for name, x, y in zip(("means", "covariances", "harmonics", "opacities"), la, lb):
        rel = float((x.grad - y.grad).norm() / y.grad.norm())
        print(f"[lpips e2e] d{name}: |fused - torch head| / |torch head| {rel:.2e}")
        assert float(y.grad.norm()) > 0 and rel <= 1e-4, (name, rel)


def test_compute_lpips_is_the_metric(monkeypatch):
    from pixelsplat_b200 import loss as L
    m = _module(4)
    monkeypatch.setattr(L, "_LPIPS_BY_DEVICE", {torch.device(DEV): m})
    a, b = _images(3, 64, 64, seed=10)
    m.train()                                                # the metric runs in eval mode regardless
    bg = b.clone().requires_grad_(True)
    got = L.compute_lpips(a, bg)
    m.eval()
    assert got.shape == (3,) and got.dtype == torch.float32 and not got.requires_grad
    assert torch.equal(got, m(a, b, normalize=True)[:, 0, 0, 0])
