"""GPU tests of the crop shim kernel (csrc/image_resample.cu through pixelsplat_b200.data.crop_shim):
PIL.Image.resize(..., Image.LANCZOS) bit for bit over the CPU tests' size grid, batched with mixed flip flags and
cropped; the float drop-ins against the reference's float route (restated here with PIL); rejected descriptors
enqueue nothing; a graph-captured device_shim replays to the same bits."""
import ctypes

import numpy as np
import pytest
import torch
from PIL import Image

from pixelsplat_b200.data import crop_shim as cs
from tests.test_crop_shim_cpu import SIZES

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _pil(img: np.ndarray, h: int, w: int) -> np.ndarray:
    return np.array(Image.fromarray(np.ascontiguousarray(img)).resize((w, h), Image.LANCZOS))


@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0][0]}x{s[0][1]}-{s[1][0]}x{s[1][1]}")
def test_kernel_equals_pil(size):
    (h, w), (ho, wo) = size
    imgs = np.random.default_rng(h * 7 + w).integers(0, 256, (4, h, w, 3), dtype=np.uint8)
    flip = torch.tensor([0, 1, 1, 0], dtype=torch.uint8, device=DEV)
    want = np.stack([_pil(im[:, ::-1] if f else im, ho, wo) for im, f in zip(imgs, flip.tolist())])
    x = torch.from_numpy(imgs).to(DEV)
    got = cs.resample_u8(x, (ho, wo), (0, 0, ho, wo), flip)
    u = (got.double() * 255).round()
    assert torch.equal(got, (u / 255).float())                    # exactly u / 255
    assert np.array_equal(u.to(torch.uint8).permute(0, 2, 3, 1).cpu().numpy(), want)
    r, c, hc, wc = (ho - (ho + 2) // 3) // 2, (wo - (wo + 2) // 3) // 2, (ho + 2) // 3, (wo + 2) // 3
    crop = cs.resample_u8(x, (ho, wo), (r, c, hc, wc), flip)
    assert torch.equal(crop, got[:, :, r:r + hc, c:c + wc])
    assert torch.equal(cs.resample_u8(x, (ho, wo), (0, 0, ho, wo), None), cs.resample_u8(
        x, (ho, wo), (0, 0, ho, wo), torch.zeros(4, dtype=torch.uint8, device=DEV)))


def _reference_rescale_and_crop(images: torch.Tensor, intrinsics: torch.Tensor, shape):
    """The reference's rescale_and_crop (src/dataset/shims/crop_shim.py), one image at a time through PIL."""
    *batch, c, h, w = images.shape
    h_out, w_out = shape
    sf = max(h_out / h, w_out / w)
    hs, ws = round(h * sf), round(w * sf)
    out = []
    for im in images.reshape(-1, c, h, w).cpu():
        u = (im * 255).clip(min=0, max=255).type(torch.uint8).permute(1, 2, 0).numpy()
        r = np.array(Image.fromarray(u).resize((ws, hs), Image.LANCZOS)) / 255
        out.append(torch.tensor(r, dtype=im.dtype).permute(2, 0, 1))
    out = torch.stack(out).reshape(*batch, c, hs, ws)
    row, col = (hs - h_out) // 2, (ws - w_out) // 2
    K = intrinsics.clone().cpu()
    K[..., 0, 0] *= ws / w_out
    K[..., 1, 1] *= hs / h_out
    return out[..., row:row + h_out, col:col + w_out], K


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("shape", [(256, 256), (180, 320), (101, 97)])
def test_float_drop_ins_match_the_reference_route(shape, dtype):
    g = torch.Generator().manual_seed(shape[0])
    images = (torch.rand(2, 3, 3, 360, 640, generator=g) * 1.2 - 0.1).to(dtype)   # out-of-range values clip
    K = torch.rand(2, 3, 3, 3, generator=g)
    want, want_K = _reference_rescale_and_crop(images, K, shape)
    got, got_K = cs.rescale_and_crop(images.to(DEV), K.to(DEV), shape)
    assert got.dtype == dtype and torch.equal(got.cpu(), want) and torch.equal(got_K.cpu(), want_K)
    ex = {"context": {"image": images[:, :2].to(DEV), "intrinsics": K[:, :2].to(DEV), "near": 1},
          "target": {"image": images[:, 2:].to(DEV), "intrinsics": K[:, 2:].to(DEV)}, "scene": ["a", "b"]}
    out = cs.apply_crop_shim(ex, shape)
    assert torch.equal(out["context"]["image"].cpu(), want[:, :2]) and out["context"]["near"] == 1
    assert torch.equal(out["target"]["intrinsics"].cpu(), want_K[:, 2:]) and out["scene"] == ["a", "b"]
    one = cs.rescale(images[0, 0].to(DEV), (60, 100))
    ref = torch.tensor(np.array(Image.fromarray(
        (images[0, 0] * 255).clip(0, 255).type(torch.uint8).permute(1, 2, 0).numpy()).resize(
        (100, 60), Image.LANCZOS)) / 255, dtype=dtype).permute(2, 0, 1)
    assert torch.equal(one.cpu(), ref)
    cropped, cK = cs.center_crop(want.to(DEV), want_K.to(DEV), (shape[0] // 2, shape[1] // 2))
    assert cropped.shape[-2:] == (shape[0] // 2, shape[1] // 2) and cK.shape == want_K.shape


def test_bad_descriptors_enqueue_nothing():
    from pixelsplat_b200 import _lib
    x = torch.zeros(2, 36, 64, 3, dtype=torch.uint8, device=DEV)
    bh, wh = cs._device_table(64, 32, 0, 32, x.device)
    bv, wv = cs._device_table(36, 18, 0, 18, x.device)
    out = torch.full((2, 3, 18, 32), -1.0, device=DEV)
    good = dict(n_images=2, in_h=36, in_w=64, out_h=18, out_w=32, taps_h=wh.shape[1], taps_v=wv.shape[1],
                images=x.data_ptr(), flip=0, bounds_h=bh.data_ptr(), weights_h=wh.data_ptr(),
                bounds_v=bv.data_ptr(), weights_v=wv.data_ptr())
    for bad in (dict(out_h=40), dict(out_w=70), dict(taps_h=65), dict(taps_v=0), dict(bounds_v=0),
                dict(images=0), dict(n_images=0)):
        before = _lib.lib.ps_launch_count()
        rc = _lib.lib.ps_image_resample(ctypes.byref(_lib.ResampleDesc(*{**good, **bad}.values())), out.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream)
        assert rc == 1 and _lib.lib.ps_launch_count() == before, bad
    torch.cuda.synchronize()
    assert (out == -1).all()
    with pytest.raises(ValueError, match="larger"):
        cs.rescale_and_crop_u8(x, torch.eye(3, device=DEV).expand(2, 3, 3), (40, 64))
    with pytest.raises(ValueError, match="uint8"):
        cs.resample_u8(x.float(), (18, 32), (0, 0, 18, 32))


def _batch(device):
    g = torch.Generator().manual_seed(3)
    u8 = lambda *s: torch.randint(0, 256, s, generator=g, dtype=torch.uint8)
    views = lambda v: {"image": u8(2, v, 360, 640, 3), "intrinsics": torch.rand(2, v, 3, 3, generator=g),
                       "extrinsics": torch.rand(2, v, 4, 4, generator=g), "near": torch.ones(2, v),
                       "far": torch.ones(2, v), "index": torch.arange(v).expand(2, v)}
    b = {"context": views(2), "target": views(3), "scene": ["a", "b"], "flip": torch.tensor([True, False])}
    if device is not None:
        b = {k: ({kk: vv.to(device) for kk, vv in v.items()} if isinstance(v, dict) else
                 v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in b.items()}
    return b


def test_device_shim_layout_and_graph_replay():
    host = _batch(None)
    out = cs.device_shim(host, (256, 256))
    assert set(out) == {"context", "target", "scene"} and out["scene"] == ["a", "b"]
    assert out["context"]["image"].shape == (2, 2, 3, 256, 256) and out["target"]["image"].shape == (2, 3, 3, 256, 256)
    for v in ("context", "target"):
        im, K = cs.rescale_and_crop_u8(host[v]["image"].to(DEV), host[v]["intrinsics"].to(DEV), (256, 256),
                                       host["flip"].to(DEV)[:, None])
        assert torch.equal(out[v]["image"], im) and torch.equal(out[v]["intrinsics"], K)
        assert torch.equal(out[v]["extrinsics"].cpu(), host[v]["extrinsics"]) and out[v]["index"].is_cuda
    # flip: image 0 is the mirror image of the unflipped shim of the same bytes (the crop is centred, 455 wide)
    ref = _pil(host["context"]["image"][0, 0].numpy()[:, ::-1], 256, 455)[:, 99:355]
    assert np.array_equal((out["context"]["image"][0, 0] * 255).round().byte().permute(1, 2, 0).cpu().numpy(), ref)

    dev = _batch(DEV)
    eager = cs.device_shim(dev, (256, 256))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        cs.device_shim(dev, (256, 256))                       # warm-up: the tables are on the device
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = cs.device_shim(dev, (256, 256))
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for v in ("context", "target"):
            assert torch.equal(captured[v]["image"], eager[v]["image"])
            assert torch.equal(captured[v]["intrinsics"], eager[v]["intrinsics"])
