"""CPU tests of SSIM: the two oracle restatements of the reference's compute_ssim (oracle/ssim_oracle.py) against
each other, scipy's filter and known answers; the torch oracle's gradient; the C ABI's and the Python layer's
argument checks (which reject before anything reaches a device)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ssim_oracle as so


def _pairs():
    rng = np.random.default_rng(5)
    yield "noise", rng.random((3, 40, 37)), rng.random((3, 40, 37))
    yy, xx = np.mgrid[0:33, 0:50] / 20.0
    smooth = 0.5 + 0.3 * np.sin(3 * xx) * np.cos(2 * yy)
    yield "smooth", smooth[None] + 0.01 * rng.standard_normal((2, 33, 50)), smooth[None] + 0.01 * rng.standard_normal(
        (2, 33, 50))
    yield "flat_bright", 0.95 + 0.002 * (2 * rng.random((1, 24, 24)) - 1), 0.95 + 0.002 * (2 * rng.random((1, 24, 24)) - 1)
    yield "above_one", 1.5 * rng.random((2, 11, 19)), 1.2 * rng.random((2, 11, 19))


def test_taps_match_the_closed_form():
    g = so.gaussian_taps()
    k = np.arange(-5, 6)
    want = np.exp(-k ** 2 / 4.5)
    assert g.shape == (11,) and abs(g.sum() - 1.0) < 1e-15
    np.testing.assert_allclose(g, want / want.sum(), rtol=0, atol=1e-16)
    assert int(3.5 * 1.5 + 0.5) == so.RADIUS


def test_numpy_filter_equals_scipy():
    nd = pytest.importorskip("scipy.ndimage")
    rng = np.random.default_rng(1)
    for shape in ((11, 11), (20, 33), (64, 13)):
        a = rng.random(shape)
        ref = nd.gaussian_filter(a, sigma=1.5, truncate=3.5, mode="reflect")
        assert np.abs(so.gaussian_filter(a) - ref).max() <= 1e-12


@pytest.mark.parametrize("case", [c[0] for c in _pairs()])
def test_the_two_restatements_agree(case):
    _, x, y = next(c for c in _pairs() if c[0] == case)
    a = so.ssim_planes_numpy(x, y)
    b = so.ssim_planes_torch(torch.from_numpy(x), torch.from_numpy(y)).numpy()
    assert np.abs(a - b).max() <= 1e-12, (a, b)
    # a float32 evaluation of the same formula drifts, but not far
    assert np.abs(so.ssim_planes_numpy(x.astype(np.float32), y.astype(np.float32), np.float32) - a).max() < 1e-4


def test_known_answers():
    rng = np.random.default_rng(2)
    x = rng.random((2, 30, 21))
    np.testing.assert_allclose(so.ssim_planes_numpy(x, x), 1.0, rtol=0, atol=1e-14)
    for a, b in ((0.2, 0.7), (1.3, 0.9), (0.0, 0.5)):
        want = (2 * a * b + so.C1) / (a * a + b * b + so.C1)
        got = so.ssim_planes_numpy(np.full((15, 12), a), np.full((15, 12), b))
        assert abs(got - want) <= 1e-12, (a, b, got, want)
        got_t = float(so.ssim_planes_torch(torch.full((15, 12), a, dtype=torch.float64),
                                           torch.full((15, 12), b, dtype=torch.float64)))
        assert abs(got_t - want) <= 1e-12
    # the image score is the channel mean
    y = rng.random((2, 30, 21))
    np.testing.assert_allclose(so.ssim_numpy(x[None], y[None]), so.ssim_planes_numpy(x, y).mean()[None], atol=1e-15)
    with pytest.raises(ValueError):
        so.ssim_planes_numpy(np.zeros((10, 10)), np.zeros((10, 10)))


def test_torch_oracle_gradcheck():
    g = torch.Generator().manual_seed(3)
    x = torch.rand((2, 13, 12), generator=g, dtype=torch.float64).requires_grad_(True)
    y = torch.rand((2, 13, 12), generator=g, dtype=torch.float64).requires_grad_(True)
    assert torch.autograd.gradcheck(so.ssim_planes_torch, (x, y), eps=1e-6, atol=1e-8)


def test_abi_rejects_invalid_arguments():
    from pixelsplat_b200 import _lib
    lib = _lib.lib
    size = ctypes.c_size_t()
    assert lib.ps_ssim_workspace_bytes(3, 11, 11, ctypes.byref(size)) == 0 and size.value >= 3 * 4
    assert size.value % 256 == 0
    assert lib.ps_ssim_workspace_bytes(96, 256, 256, ctypes.byref(size)) == 0
    assert size.value >= 96 * 8 * 8 * 4                 # one partial per 16 x 32 tile of the 246 x 246 crop
    for n, h, w in ((0, 64, 64), (-1, 64, 64), (1, 10, 64), (1, 64, 10), (1, 0, 0)):
        assert lib.ps_ssim_workspace_bytes(n, h, w, ctypes.byref(size)) == 1
        assert b"bad shape" in lib.ps_last_error()
    assert lib.ps_ssim_workspace_bytes(1, 64, 64, None) == 1
    lib.ps_ssim_workspace_bytes(2, 64, 64, ctypes.byref(size))
    ws_bytes = size.value
    # dummy (host) addresses: every call below must fail validation before touching them
    bufs = [ctypes.create_string_buffer(16) for _ in range(6)]
    p = [ctypes.addressof(b) for b in bufs]
    fwd = lambda n, h, w, x, y, o, ws, wb: lib.ps_ssim_forward(n, h, w, x, y, o, ws, wb, None)
    assert fwd(0, 64, 64, p[0], p[1], p[2], p[3], ws_bytes) == 1
    assert fwd(2, 10, 64, p[0], p[1], p[2], p[3], ws_bytes) == 1
    assert fwd(2, 64, 10, p[0], p[1], p[2], p[3], ws_bytes) == 1
    for i in range(4):
        args = p[:4]
        args[i] = None
        assert fwd(2, 64, 64, *args, ws_bytes) == 1 and b"NULL" in lib.ps_last_error()
    assert fwd(2, 64, 64, p[0], p[1], p[2], p[3], ws_bytes - 1) == 1 and b"workspace" in lib.ps_last_error()
    bwd = lambda n, h, w, x, y, d, dx, dy, ws, wb: lib.ps_ssim_backward(n, h, w, x, y, d, dx, dy, ws, wb, None)
    assert bwd(0, 64, 64, *p, ws_bytes) == 1
    assert bwd(2, 10, 64, *p, ws_bytes) == 1
    assert bwd(2, 64, 10, *p, ws_bytes) == 1
    for i in (0, 1, 2, 4, 5):                           # d_x (index 3) may be NULL
        args = list(p)
        args[i] = None
        assert bwd(2, 64, 64, *args, ws_bytes) == 1 and b"NULL" in lib.ps_last_error()
    assert bwd(2, 64, 64, *p, ws_bytes - 1) == 1 and b"workspace" in lib.ps_last_error()


def test_python_layer_rejects_invalid_inputs():
    from pixelsplat_b200.loss import compute_ssim, ssim
    a = torch.rand(2, 3, 32, 32)
    with pytest.raises(ValueError, match="no CPU path"):
        ssim(a, a.clone())
    with pytest.raises(ValueError, match="float32"):
        ssim(a.double(), a.double())
    with pytest.raises(ValueError, match="float32"):
        ssim(a.half(), a.half())
    with pytest.raises(ValueError, match="one shape"):
        ssim(a, a[:, :, :31])
    with pytest.raises(ValueError, match="one shape"):
        ssim(a[0], a[0])
    with pytest.raises(ValueError, match="at least 11"):
        ssim(torch.rand(1, 3, 10, 10), torch.rand(1, 3, 10, 10))
    with pytest.raises(ValueError, match="at least 11"):
        compute_ssim(torch.rand(1, 3, 10, 40), torch.rand(1, 3, 10, 40))
