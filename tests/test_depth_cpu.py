"""CPU tests of the depth channel's host surface: the C-ABI fields (depth_mode, near_far, depth_image, run_depth,
ps_get_option, ps_raster_backward_depth), the workspace sizes with and without depth, and the LossDepth drop-in
against the reference module's golden output."""
import ctypes
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
HEADER = ROOT / "include" / "pixelsplat_b200.h"


def loss_depth_case(dtype=torch.float64, b: int = 2, v: int = 2, h: int = 12, w: int = 14) -> dict:
    """Inputs of the LossDepth fixture (tests/golden/loss_depth.npz, regenerated on both sides): a log-depth map that
    crosses both clamps, per-view near / far and a ground-truth image with edges."""
    from tests.golden_util import seeded_like
    near = 0.5 + 0.5 * seeded_like("loss_depth.near", (b, v)).abs()
    far = near + 5.0 + seeded_like("loss_depth.far", (b, v)).abs()
    depth = 0.2 + 0.9 * seeded_like("loss_depth.depth", (b, v, h, w))
    image = torch.sigmoid(2.0 * seeded_like("loss_depth.image", (b, v, 3, h, w)))
    return {k: t.to(dtype) for k, t in dict(depth=depth, near=near, far=far, image=image).items()}


def test_depth_fields_match_the_header(tmp_path):
    from pixelsplat_b200 import _lib
    fields = ("offsetof(ps_raster_desc,depth_mode)", "offsetof(ps_raster_desc,sh_basis)",
              "offsetof(ps_raster_inputs,near_far)", "offsetof(ps_raster_layout,depth_image)",
              "offsetof(ps_raster_layout,run_depth)", "sizeof(ps_raster_desc)", "sizeof(ps_raster_inputs)",
              "sizeof(ps_raster_layout)", "PS_DEPTH_NONE", "PS_DEPTH_Z", "PS_DEPTH_DISPARITY",
              "PS_DEPTH_RELATIVE_DISPARITY", "PS_DEPTH_LOG")
    probe = tmp_path / "probe.c"
    probe.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "pixelsplat_b200.h"\n'
                     "int main(void){" + "".join(f'printf("%zu\\n",(size_t)({f}));' for f in fields) + "return 0;}\n")
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", str(HEADER.parent), str(probe), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    want = [_lib.RasterDesc.depth_mode.offset, _lib.RasterDesc.sh_basis.offset, _lib.RasterInputs.near_far.offset,
            _lib.RasterLayout.depth_image.offset, _lib.RasterLayout.run_depth.offset, ctypes.sizeof(_lib.RasterDesc),
            ctypes.sizeof(_lib.RasterInputs), ctypes.sizeof(_lib.RasterLayout)] + [
        _lib.DEPTH_MODES[m] for m in (None, "depth", "disparity", "relative_disparity", "log")]
    assert got == want
    # the descriptor keeps its size and offsets: depth_mode took the place of the reserved word
    assert ctypes.sizeof(_lib.RasterDesc) == 64 and _lib.RasterDesc.depth_mode.offset == 60
    # the new entry points are bound
    assert _lib.lib.ps_raster_backward_depth.restype is ctypes.c_int and _lib.lib.ps_get_option.restype is ctypes.c_int


def _desc(depth_mode, S=2, V=3, H=70, W=50):
    from pixelsplat_b200 import _lib
    return _lib.RasterDesc(S, V, 1000, 25, 4, _lib.PS_SH_3M, _lib.PS_COV_3X3, H, W, 0, 0, 12345, 0, depth_mode)


def test_depth_mode_is_validated():
    from pixelsplat_b200 import _lib
    for bad in (-1, 5, 1 << 20):
        with pytest.raises(ValueError, match="PS_ERR_INVALID_ARGUMENT.*bad depth_mode"):
            _lib.sizes(_desc(bad))
    for ok in range(5):
        _lib.sizes(_desc(ok))
    # NULL d_depth / a colour-only desc are rejected before anything is launched
    rc = _lib.lib.ps_raster_backward_depth(ctypes.byref(_desc(1)), None, None, None, None, None, None, None, 0,
                                           None, None)
    assert rc == 1 and b"d_depth is NULL" in _lib.lib.ps_last_error()
    buf = ctypes.c_float()
    rc = _lib.lib.ps_raster_backward_depth(ctypes.byref(_desc(0)), None, None, None, None, None, ctypes.byref(buf),
                                           None, 0, None, None)
    assert rc == 1 and b"depth_mode" in _lib.lib.ps_last_error()


def test_depth_sizes():
    """Mode 0 is today's workspace (no depth arrays); a depth mode grows only the image state, by the depth image
    and the run depths."""
    from pixelsplat_b200 import _lib
    S, V, H, W = 2, 3, 70, 50
    px = S * V * H * W
    align = lambda x: (x + 255) // 256 * 256
    s0, l0 = _lib.sizes(_desc(0)), _lib.layout(_desc(0))
    assert l0.depth_image == 0 and l0.run_depth == 0
    assert s0.image_bytes == 2 * align(px * 4) + align(px * 12) + align(px * 16 * 3)
    for mode in range(1, 5):
        s1, l1 = _lib.sizes(_desc(mode)), _lib.layout(_desc(mode))
        assert (s1.geom_bytes, s1.binning_bytes, s1.backward_bytes) == (s0.geom_bytes, s0.binning_bytes,
                                                                        s0.backward_bytes)
        assert s1.image_bytes - s0.image_bytes >= px * 4 + 3 * px * 4
        assert l1.depth_image >= s0.image_bytes - 255 and l1.run_depth - l1.depth_image >= px * 4
        assert l1.run_depth + 3 * px * 4 <= s1.image_bytes
        assert all(getattr(l1, f) == getattr(l0, f) for f, _ in _lib.RasterLayout._fields_[:-2])


def test_get_option_round_trip():
    from pixelsplat_b200 import _lib
    try:
        for name, values in (("composite_impl", (1, 2)), ("composite_segments", (0, 1, 2, 4)),
                             ("composite_hit_lists", (0, 1, 2))):
            for v in values:
                _lib.set_option(name, v)
                assert _lib.get_option(name) == v
        with pytest.raises(ValueError, match="unknown option"):
            _lib.get_option("composite_depth")
    finally:
        _lib.set_option("composite_impl", 2)
        _lib.set_option("composite_segments", 0)
        _lib.set_option("composite_hit_lists", 2)
    assert [_lib.get_option(n) for n in ("composite_impl", "composite_segments", "composite_hit_lists")] == [2, 0, 2]


def test_get_option_sees_the_environment():
    """A compositor chosen through PIXELSPLAT_B200_COMPOSITE is what ps_get_option reports."""
    import os
    import sys
    env = dict(os.environ, PIXELSPLAT_B200_COMPOSITE="1", PIXELSPLAT_B200_SEGMENTS="2")
    code = ("from pixelsplat_b200 import _lib; from pixelsplat_b200.decoder import cuda_splatting as c; "
            "print(_lib.get_option('composite_impl'), _lib.get_option('composite_segments'), c._legacy_compositor())")
    r = subprocess.run([sys.executable, "-c", code], cwd=str(ROOT), env=env, capture_output=True, text=True,
                       check=True)
    assert r.stdout.split() == ["1", "2", "True"]


@pytest.mark.parametrize("sigma", [None, 12.0])
@pytest.mark.parametrize("second", [False, True])
def test_loss_depth_matches_the_reference_golden(sigma, second):
    """pixelsplat_b200.loss.LossDepth against the reference's LossDepth (tests/golden/loss_depth.npz, written by
    oracle/make_loss_depth_golden.py): loss value and gradient w.r.t. the depth map, float64 and float32."""
    from pixelsplat_b200 import loss as L
    gold = np.load(ROOT / "tests" / "golden" / "loss_depth.npz")
    for dtype, tag, tol in ((torch.float64, "f64", 1e-12), (torch.float32, "f32", 1e-6)):
        c = loss_depth_case(dtype)
        depth = c["depth"].clone().requires_grad_(True)
        m = L.LossDepth(L.LossDepthCfgWrapper(L.LossDepthCfg(0.25, sigma, second)))
        assert m.name == "depth"
        out = m(type("O", (), {"depth": depth})(), {"target": {"near": c["near"], "far": c["far"],
                                                              "image": c["image"]}})
        out.backward()
        out = out.detach()
        key = f"{tag}_{'none' if sigma is None else int(sigma)}_{int(second)}"
        ref_loss, ref_grad = gold[key + "_loss"], gold[key + "_grad"]
        assert abs(float(out) - float(ref_loss)) <= tol * abs(float(ref_loss)), (key, float(out), float(ref_loss))
        g = depth.grad.numpy()
        assert np.abs(g - ref_grad).max() <= tol * np.abs(ref_grad).max(), key
        assert np.abs(ref_grad).max() > 0
