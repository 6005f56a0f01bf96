"""CPU tests of the crop shim's coefficient tables (pixelsplat_b200.data.crop_shim.resample_table): with the
integer passes of oracle/resample_oracle.py they give PIL.Image.resize(..., Image.LANCZOS) bit for bit on uniform
noise (the worst case for rounding), flipped or not, and a crop's tables give the crop of the full result.  Also
the u / 255 conversion, the reference's size arithmetic, and the C ABI's rejections (no GPU needed)."""
import ctypes

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import resample_oracle as ro
from pixelsplat_b200.data import crop_shim as cs

# (input h, w) -> (output h, w): the reference's 360 x 640 crops, one axis unchanged (that pass skipped), an
# unchanged size (a copy), odd and prime sizes
SIZES = [((360, 640), (256, 455)), ((360, 640), (180, 320)), ((50, 80), (50, 33)), ((64, 64), (17, 64)),
         ((41, 59), (41, 59)), ((97, 131), (61, 89)), ((101, 97), (53, 97)), ((127, 211), (7, 13))]


def _pil(img: np.ndarray, h: int, w: int) -> np.ndarray:
    return np.array(Image.fromarray(img).resize((w, h), Image.LANCZOS))


@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0][0]}x{s[0][1]}-{s[1][0]}x{s[1][1]}")
def test_tables_and_integer_passes_equal_pil(size, flip):
    (h, w), (ho, wo) = size
    img = np.random.default_rng(h * 1000 + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    want = _pil(np.ascontiguousarray(img[:, ::-1]) if flip else img, ho, wo)
    got = ro.resample_and_crop(img, (ho, wo), (0, 0, ho, wo), flip)
    assert np.array_equal(got, want), f"{int((got != want).sum())} bytes differ"
    r, c = (ho - (ho + 1) // 2) // 2, (wo - (wo + 1) // 2) // 2
    crop = ro.resample_and_crop(img, (ho, wo), (r, c, (ho + 1) // 2, (wo + 1) // 2), flip)
    assert np.array_equal(crop, want[r:r + (ho + 1) // 2, c:c + (wo + 1) // 2])


def test_skipped_axis_is_the_identity_table():
    b, w = cs.resample_table(64, 64, 5, 10)
    assert w.shape == (10, 1) and (w == 1 << 22).all() and (b[:, 0] == np.arange(5, 15)).all() and (b[:, 1] == 1).all()
    b, w = cs.resample_table(640, 455)
    assert b.shape == (455, 2) and w.shape[1] == b[:, 1].max() and (w.sum(1) > 0).all()
    assert b[:, 0].min() >= 0 and (b[:, 0] + b[:, 1]).max() <= 640


def test_table_rejects_bad_sizes():
    for args in ((10, 11, 0, None), (10, 5, 3, 3), (10, 0, 0, None), (10, 5, -1, 2)):
        with pytest.raises(ValueError):
            cs.resample_table(*args)


def test_u_over_255_is_the_reference_conversion():
    u = np.arange(256, dtype=np.uint8)
    ref = torch.tensor(u / 255, dtype=torch.float32)                     # np.array(img) / 255, then float32
    ours = torch.from_numpy(u.astype(np.float32)) / 255.0                # the kernel's (float)u / 255.0f
    assert torch.equal(ref, ours)
    back = (ref * 255).clip(min=0, max=255).type(torch.uint8)           # the reference's float -> uint8
    assert torch.equal(back, torch.from_numpy(u))


def test_scaled_shape_follows_the_reference():
    assert cs.scaled_shape(360, 640, (256, 256)) == (256, 455)
    assert cs.scaled_shape(360, 640, (180, 320)) == (180, 320)
    with pytest.raises(ValueError):
        cs.scaled_shape(100, 100, (200, 50))


def test_cpu_tensors_raise():
    img = torch.rand(2, 3, 36, 64)
    K = torch.eye(3).expand(2, 3, 3)
    with pytest.raises(ValueError, match="CUDA"):
        cs.rescale_and_crop(img, K, (18, 32))
    with pytest.raises(ValueError, match="CUDA"):
        cs.rescale(img[0], (18, 32))
    with pytest.raises(ValueError, match="CUDA"):
        cs.center_crop(img, K, (18, 32))
    with pytest.raises(ValueError, match="CUDA"):
        cs.rescale_and_crop_u8(torch.zeros(2, 36, 64, 3, dtype=torch.uint8), K, (18, 32))


def _desc(**kw):
    from pixelsplat_b200 import _lib
    d = dict(n_images=2, in_h=36, in_w=64, out_h=18, out_w=32, taps_h=5, taps_v=5, images=16, flip=0,
             bounds_h=16, weights_h=16, bounds_v=16, weights_v=16)
    d.update(kw)
    return _lib.ResampleDesc(*d.values())


@pytest.mark.parametrize("bad", [dict(n_images=0), dict(n_images=70000), dict(out_h=37), dict(out_w=65),
                                 dict(in_h=0), dict(taps_h=0), dict(taps_h=65), dict(taps_v=37), dict(images=0),
                                 dict(bounds_h=0), dict(weights_v=0)], ids=lambda b: "-".join(map(str, b.items())))
def test_abi_rejects_bad_descriptors(bad):
    from pixelsplat_b200 import _lib
    before = _lib.lib.ps_launch_count()
    rc = _lib.lib.ps_image_resample(ctypes.byref(_desc(**bad)), ctypes.c_void_p(16), None)
    assert rc == 1 and _lib.lib.ps_launch_count() == before
    assert b"ps_image_resample" in _lib.lib.ps_last_error()
    assert _lib.lib.ps_image_resample(None, ctypes.c_void_p(16), None) == 1
    assert _lib.lib.ps_image_resample(ctypes.byref(_desc()), None, None) == 1
