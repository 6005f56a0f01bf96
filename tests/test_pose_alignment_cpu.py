"""CPU side of test-time pose alignment: the twist parameterisation of pixelsplat_b200.pose against float64 central
differences and the matrix exponential, and the C ABI rules of the camera-only backward (ps_raster_grads with every
Gaussian output NULL), checked without a GPU."""
import ctypes

import pytest
import torch

from pixelsplat_b200.pose import apply_twists, twist_to_transform


def _central(f, x, h):
    cols = []
    for i in range(x.numel()):
        xp, xm = x.clone(), x.clone()
        xp.view(-1)[i] += h
        xm.view(-1)[i] -= h
        cols.append(((f(xp) - f(xm)) / (2 * h)).reshape(-1))
    return torch.stack(cols, -1)          # [outputs, inputs]


TWISTS = [
    [0.0, 0.0, 0.0, 0.0, 0.0, 0.0],                  # the starting point of every alignment (Taylor branch)
    [3e-5, -2e-5, 1e-5, 0.01, 0.0, -0.02],           # |omega|^2 < 1e-8: still the Taylor branch
    [0.03, -0.04, 0.02, 0.02, -0.015, 0.01],         # ~3 degrees
    [0.9, 0.4, -1.2, 0.3, -0.2, 0.5],                # large
]


@pytest.mark.parametrize("xi", TWISTS)
def test_twist_derivative_matches_central_differences(xi):
    x = torch.tensor(xi, dtype=torch.float64)
    jac = torch.autograd.functional.jacobian(lambda t: twist_to_transform(t).reshape(-1), x)
    fd = _central(lambda t: twist_to_transform(t), x, 1e-6)
    assert torch.isfinite(jac).all()
    assert torch.allclose(jac, fd, rtol=1e-6, atol=1e-8), float((jac - fd).abs().max())


@pytest.mark.parametrize("xi", TWISTS)
def test_twist_is_the_exponential_map_of_the_rotation(xi):
    x = torch.tensor(xi, dtype=torch.float64)
    T = twist_to_transform(x)
    w = x[:3]
    W = torch.tensor([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]], dtype=torch.float64)
    assert torch.allclose(T[:3, :3], torch.linalg.matrix_exp(W), rtol=0, atol=1e-14)
    assert torch.equal(T[:3, 3], x[3:]) and torch.equal(T[3], torch.tensor([0.0, 0.0, 0.0, 1.0], dtype=torch.float64))
    assert torch.allclose(T[:3, :3] @ T[:3, :3].T, torch.eye(3, dtype=torch.float64), atol=1e-14)


def test_twists_apply_in_the_camera_frame_and_batch():
    g = torch.Generator().manual_seed(0)
    xi = 0.1 * torch.randn(2, 3, 6, generator=g, dtype=torch.float64)
    E = twist_to_transform(torch.randn(2, 3, 6, generator=g, dtype=torch.float64))
    out = apply_twists(E, xi)
    for s in range(2):
        for v in range(3):
            assert torch.allclose(out[s, v], E[s, v] @ twist_to_transform(xi[s, v]), atol=1e-15)
    # a pure translation twist moves the camera centre along its own axes
    t = torch.tensor([0.0, 0.0, 0.0, 0.1, 0.2, 0.3], dtype=torch.float64)
    moved = apply_twists(E[0, 0], t)
    assert torch.allclose(moved[:3, 3], E[0, 0, :3, 3] + E[0, 0, :3, :3] @ t[3:], atol=1e-15)


def _abi():
    from pixelsplat_b200 import _lib
    d = _lib.RasterDesc(1, 2, 100, 25, 4, 0, 0, 16, 16, 0, 0, 1000)
    sz = _lib.sizes(d)
    ins = _lib.RasterInputs(*([1 << 20] * 9), None, None)
    st = _lib.RasterState(1 << 20, sz.geom_bytes, 1 << 20, sz.binning_bytes, 1 << 20, sz.image_bytes)
    return _lib, d, sz, ins, st


def _backward(lib, d, sz, ins, st, grads):
    fake = ctypes.c_void_p(1 << 20)
    return lib.ps_raster_backward(ctypes.byref(d), ctypes.byref(ins), ctypes.byref(st), fake, fake,
                                  sz.backward_bytes, ctypes.byref(grads), None)


def test_camera_only_backward_argument_rules_without_gpu():
    _lib, d, sz, ins, st = _abi()
    lib = _lib.lib
    need = _lib.camera_workspace_bytes(d)
    P = 1 << 20
    # every Gaussian output NULL and no camera gradients: nothing to compute
    grads = _lib.RasterGrads(None, None, None, None, None, None)
    assert _backward(lib, d, sz, ins, st, grads) == 1
    assert b"no camera gradients" in lib.ps_last_error()
    cam = _lib.RasterCameraGrads(P, None, None, None, P, need)
    # some but not all of the Gaussian outputs NULL, with and without camera gradients
    for camera in (None, ctypes.pointer(cam)):
        for i in range(4):
            ptrs = [P, P, P, P, None]
            ptrs[i] = None
            assert _backward(lib, d, sz, ins, st, _lib.RasterGrads(*ptrs, camera)) == 1, (i, camera)
            assert b"required gradient pointer" in lib.ps_last_error()
        # only means2d given
        assert _backward(lib, d, sz, ins, st, _lib.RasterGrads(None, None, None, None, P, camera)) == 1
        assert b"required gradient pointer" in lib.ps_last_error()
    # the camera-only form passes the pointer rules and meets the same workspace checks as the full backward
    for ws, nbytes in ((None, need), (P, need - 1), (P + 4, need)):
        cam = _lib.RasterCameraGrads(P, None, None, None, ws, nbytes)
        grads = _lib.RasterGrads(None, None, None, None, None, ctypes.pointer(cam))
        assert _backward(lib, d, sz, ins, st, grads) == 1
        assert b"camera-gradient workspace" in lib.ps_last_error()
    # the other backward entry points apply the same rules
    fake = ctypes.c_void_p(P)
    grads = _lib.RasterGrads(None, None, None, None, None, None)
    rc = lib.ps_raster_backward_loss(ctypes.byref(d), ctypes.byref(ins), ctypes.byref(st), fake, fake, fake,
                                     sz.backward_bytes, ctypes.byref(grads), None)
    assert rc == 1 and b"no camera gradients" in lib.ps_last_error()
