"""CPU side of the camera gradients: the function they differentiate is pinned (float64 autograd of the
rasterizer restatement and of the camera set-up chain against central differences), and the C ABI of
ps_raster_camera_grads / ps_camera_setup_backward is checked without a GPU."""
import ctypes
import subprocess
from pathlib import Path

import pytest
import torch

from tests.camera_grads_f64 import camera_chain, render_view

ROOT = Path(__file__).resolve().parents[1]
HEADER = ROOT / "include" / "pixelsplat_b200.h"


def _small_scene(seed=0, p=6, use_sh=True):
    """A few Gaussians well inside a 32x32 view: opacity <= 0.5 (T stays far above 1e-4), screen sizes of a few
    pixels, no clamp."""
    g = torch.Generator().manual_seed(seed)
    z = 3.0 + 2.0 * torch.rand(p, generator=g, dtype=torch.float64)
    uv = 0.3 + 0.4 * torch.rand(p, 2, generator=g, dtype=torch.float64)
    means = torch.cat([(uv - 0.5) / 0.88 * z[:, None], z[:, None]], -1)
    a = 0.05 * torch.randn(p, 3, 3, generator=g, dtype=torch.float64)
    cov = a @ a.transpose(1, 2) + 0.004 * torch.eye(3, dtype=torch.float64)
    row, col = torch.triu_indices(3, 3)
    cov6 = cov[:, row, col]
    opac = 0.2 + 0.3 * torch.rand(p, generator=g, dtype=torch.float64)
    sh = 0.3 * torch.randn(p, 9, 3, generator=g, dtype=torch.float64) if use_sh else None
    colors = None if use_sh else torch.rand(p, 3, generator=g, dtype=torch.float64)
    ext = torch.eye(4, dtype=torch.float64)
    ext[:3, 3] = torch.tensor([0.05, -0.03, 0.1], dtype=torch.float64)
    K = torch.tensor([[0.88, 0.0, 0.5], [0.0, 0.9, 0.48], [0.0, 0.0, 1.0]], dtype=torch.float64)
    return means, cov6, opac, sh, colors, ext, K


def _central(f, x, h):
    out = torch.zeros_like(x)
    flat = out.view(-1)
    for i in range(x.numel()):
        xp, xm = x.clone(), x.clone()
        xp.view(-1)[i] += h
        xm.view(-1)[i] -= h
        flat[i] = (f(xp) - f(xm)) / (2 * h)
    return out


@pytest.mark.parametrize("use_sh,depth_mode", [(True, None), (False, None), (True, "depth"), (True, "disparity")])
def test_raster_camera_gradients_match_central_differences(use_sh, depth_mode):
    means, cov6, opac, sh, colors, ext, K = _small_scene(use_sh=use_sh)
    W = H = 32
    vm, pm, campos, tanfov, _ = camera_chain(ext, K, 0.5, 100.0, scale_invariant=False)
    vm, pm, campos, tanfov = (t.detach().clone() for t in (vm, pm, campos, tanfov))
    g = torch.Generator().manual_seed(1)
    dC = torch.randn(3, H, W, generator=g, dtype=torch.float64)
    dD = torch.randn(H, W, generator=g, dtype=torch.float64)
    bg = torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64)

    def loss(vm_, pm_, cp_, tf_):
        c, d = render_view(means, cov6, opac, sh, colors, vm_, pm_, cp_, tf_, bg, W, H, 2,
                           depth_mode=depth_mode, near=0.5, far=100.0)
        out = (c * dC).sum()
        return out if d is None else out + (d * dD).sum()

    leaves = [t.clone().requires_grad_(True) for t in (vm, pm, campos, tanfov)]
    loss(*leaves).backward()
    base = [vm, pm, campos, tanfov]
    for i, leaf in enumerate(leaves):
        def f(x, i=i):
            args = list(base)
            args[i] = x
            return loss(*args)
        fd = _central(f, base[i], 1e-6)
        got = leaf.grad if leaf.grad is not None else torch.zeros_like(leaf)   # campos unused with colours
        assert torch.allclose(got, fd, rtol=1e-5, atol=1e-7 * max(float(fd.abs().max()), 1.0)), (i, got, fd)
    # entries the forward never reads get exact zeros; colours instead of SH give d_campos = 0
    assert (leaves[0].grad[[3, 7, 11, 15]] == 0).all() and (leaves[1].grad[[2, 6, 10, 14]] == 0).all()
    if not use_sh:
        assert leaves[2].grad is None or (leaves[2].grad == 0).all()


@pytest.mark.parametrize("scale_invariant", [True, False])
def test_camera_chain_matches_central_differences(scale_invariant):
    _, _, _, _, _, ext, K = _small_scene()
    ext = ext.clone()
    rot = torch.linalg.matrix_exp(torch.tensor([[0.0, -0.1, 0.05], [0.1, 0.0, -0.2], [-0.05, 0.2, 0.0]],
                                               dtype=torch.float64))
    ext[:3, :3] = rot
    g = torch.Generator().manual_seed(2)
    w = [torch.randn(n, generator=g, dtype=torch.float64) for n in (16, 16, 3, 2)]

    def loss(e, k):
        outs = camera_chain(e, k, 0.4, 50.0, scale_invariant)[:4]
        return sum((o * wi).sum() for o, wi in zip(outs, w))

    e, k = ext.clone().requires_grad_(True), K.clone().requires_grad_(True)
    loss(e, k).backward()
    fd_e = _central(lambda x: loss(x, K), ext, 1e-6)
    fd_k = _central(lambda x: loss(ext, x), K, 1e-6)
    assert torch.allclose(e.grad, fd_e, rtol=1e-6, atol=1e-8 * float(fd_e.abs().max()))
    assert torch.allclose(k.grad, fd_k, rtol=1e-6, atol=1e-8 * float(fd_k.abs().max()))


def test_camera_grads_structs_match_the_header(tmp_path):
    from pixelsplat_b200 import _lib
    probe = tmp_path / "probe.c"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pixelsplat_b200.h"\n'
                     'int main(void){printf("%zu %zu %zu %zu\\n", sizeof(ps_raster_camera_grads),'
                     "offsetof(ps_raster_camera_grads,workspace_bytes),sizeof(ps_raster_grads),"
                     "offsetof(ps_raster_grads,camera));return 0;}\n")
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", str(HEADER.parent), str(probe), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [ctypes.sizeof(_lib.RasterCameraGrads), _lib.RasterCameraGrads.workspace_bytes.offset,
                   ctypes.sizeof(_lib.RasterGrads), _lib.RasterGrads.camera.offset]


@pytest.mark.parametrize("S,V,P", [(1, 1, 1), (1, 1, 32), (2, 3, 1000), (4, 2, 17), (1, 4, 393216)])
def test_camera_workspace_closed_form_and_other_sizes_unchanged(S, V, P):
    from pixelsplat_b200 import _lib
    d = _lib.RasterDesc(S, V, P, 25, 4, _lib.PS_SH_3M, _lib.PS_COV_3X3, 70, 50, 0, 0, 12345)
    assert _lib.camera_workspace_bytes(d) == S * V * ((P - 1) // 32 + 2) * 128
    # at least one row for every warp of 32 consecutive (scene, Gaussian) indices that overlaps a scene
    for s in range(S):
        assert (((s + 1) * P - 1) // 32 - (s * P) // 32 + 1) <= (P - 1) // 32 + 2
    bad = _lib.RasterDesc(S, V, 0, 25, 4, 0, 0, 16, 16, 0, 0, 100)
    with pytest.raises(ValueError, match="PS_ERR_INVALID_ARGUMENT"):
        _lib.camera_workspace_bytes(bad)


def test_camera_argument_validation_without_gpu():
    from pixelsplat_b200 import _lib
    lib = _lib.lib
    fake = ctypes.c_void_p(1 << 20)
    # ps_camera_setup_backward: n < 1 and NULL required pointers
    assert lib.ps_camera_setup_backward(0, fake, fake, fake, fake, 1, None, None, None, None, fake, fake, None) == 1
    for i in range(6):
        args = [fake] * 4 + [1] + [None] * 4 + [fake, fake]
        pos = [0, 1, 2, 3, 9, 10][i]
        args[pos] = None
        assert lib.ps_camera_setup_backward(4, *args, None) == 1, i
    # a short or missing camera workspace is rejected before anything is enqueued
    d = _lib.RasterDesc(1, 2, 100, 25, 4, 0, 0, 16, 16, 0, 0, 1000)
    sz = _lib.sizes(d)
    ins = _lib.RasterInputs(*([1 << 20] * 9), None, None)
    st = _lib.RasterState(1 << 20, sz.geom_bytes, 1 << 20, sz.binning_bytes, 1 << 20, sz.image_bytes)
    need = _lib.camera_workspace_bytes(d)
    for ws, nbytes in ((None, need), (1 << 20, need - 1), ((1 << 20) + 4, need)):
        cam = _lib.RasterCameraGrads(1 << 20, None, None, None, ws, nbytes)
        grads = _lib.RasterGrads(1 << 20, 1 << 20, 1 << 20, 1 << 20, None, ctypes.pointer(cam))
        rc = lib.ps_raster_backward(ctypes.byref(d), ctypes.byref(ins), ctypes.byref(st), fake, fake,
                                    sz.backward_bytes, ctypes.byref(grads), None)
        assert rc == 1 and b"camera-gradient workspace" in lib.ps_last_error()
