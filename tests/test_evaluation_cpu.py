"""CPU tests of the evaluation (pixelsplat_b200.evaluation): the reference's PNG round trip equals
trunc(clip(x, 0, 1) * 255) / 255 (so scoring the frame pass's planes is scoring the PNGs), checkpoint loading,
the C ABI's rejections of the frame pass, and the metric computer's skipping and aggregation."""
import ctypes
import json
import pickle
from dataclasses import dataclass
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

GOLDEN = Path(__file__).resolve().parent / "golden"


# ---- the reference's image_io route, restated (PIL + numpy; its module imports matplotlib)

def ref_prep_image(image: torch.Tensor) -> np.ndarray:
    """src/misc/image_io.py prep_image for a [3, h, w] image."""
    return (image.detach().clip(min=0, max=1) * 255).type(torch.uint8).permute(1, 2, 0).cpu().numpy()


def ref_round_trip(image: torch.Tensor, path: Path) -> torch.Tensor:
    """save_image, then load_image: PNG through PIL, read back as ToTensor does (u as float32, divided by 255)."""
    Image.fromarray(ref_prep_image(image)).save(path)
    u = torch.from_numpy(np.array(Image.open(path))).permute(2, 0, 1).contiguous()
    return u.to(torch.float32).div(255)[:3]


def crafted_values() -> np.ndarray:
    """Exact k/255, k/255 one ulp either side, 0, 1, signed zeros, negatives, values above 1 and infinities."""
    k = (np.arange(256, dtype=np.float32) / np.float32(255)).astype(np.float32)
    v = np.concatenate([k, np.nextafter(k, np.float32(2)), np.nextafter(k, np.float32(-1)),
                        np.array([0.0, -0.0, 1.0, -1e-30, -0.5, -3.0, 1.0000001, 1.5, 7.0, 1e30, np.inf, -np.inf,
                                  0.5, 0.99999994, 1.0 / 510, 254.5 / 255], np.float32)])
    return v.astype(np.float32)


def crafted_image(h: int, w: int, seed: int = 0) -> torch.Tensor:
    """[3, h, w]: the crafted values (cycled, shuffled) mixed with uniform noise on [-0.1, 1.1]."""
    rng = np.random.default_rng(seed)
    v = crafted_values()
    x = rng.uniform(-0.1, 1.1, 3 * h * w).astype(np.float32)
    n = min(v.size, x.size)
    x[rng.permutation(x.size)[:n]] = rng.permutation(v)[:n]
    return torch.from_numpy(x.reshape(3, h, w))


def trunc_quantised(x: np.ndarray) -> np.ndarray:
    c = np.clip(x, np.float32(0), np.float32(1)).astype(np.float32)
    return (np.trunc(c * np.float32(255)) / np.float32(255)).astype(np.float32)


@pytest.mark.parametrize("hw", [(32, 32), (7, 13), (1, 1), (17, 31)])
def test_png_round_trip_is_truncation(tmp_path, hw):
    x = crafted_image(*hw, seed=hw[0] * 100 + hw[1])
    got = ref_round_trip(x, tmp_path / "f.png").numpy()
    assert np.array_equal(got, trunc_quantised(x.numpy()))


def test_round_trip_on_every_crafted_value(tmp_path):
    v = crafted_values()
    x = torch.from_numpy(np.stack([v, v[::-1].copy(), np.roll(v, 7)])[:, None, :])   # [3, 1, n]
    got = ref_round_trip(x, tmp_path / "f.png").numpy()
    assert np.array_equal(got, trunc_quantised(x.numpy()))
    # k/255 comes back as itself, one ulp below it truncates to (k-1)/255
    k = np.arange(1, 256)
    assert np.array_equal(got[0, 0, k], v[k]) and np.array_equal(got[0, 0, 2 * 256 + k], v[k - 1])


def test_cpu_tensors_raise():
    from pixelsplat_b200.evaluation import frame_pass, prep_image
    with pytest.raises(ValueError, match="CUDA"):
        frame_pass(torch.rand(2, 3, 8, 8))
    with pytest.raises(ValueError, match="CUDA"):
        prep_image(torch.rand(3, 8, 8))
    with pytest.raises(ValueError, match="float32 renders or uint8"):
        frame_pass(torch.rand(2, 3, 8, 8, dtype=torch.float64))


# ---- checkpoint loading

@pytest.fixture(scope="module")
def encoder():
    from pixelsplat_b200.evaluation.presets import encoder_cfg
    from pixelsplat_b200.encoder.encoder_epipolar import EncoderEpipolar
    return EncoderEpipolar(encoder_cfg("re10k"), num_context_views=2)


def _reference_state_dict():
    """The reference EncoderEpipolar's keys and shapes, filled with distinct values."""
    keys = json.loads((GOLDEN / "backbone_keys.json").read_text())["EncoderEpipolar"]
    return {k: torch.full(tuple(s), i, dtype=torch.int64) if k.endswith("num_batches_tracked")
            else torch.full(tuple(s), float(i % 89) / 89.0) for i, (k, s) in enumerate(keys)}


def _lightning(state_dict: dict, step: int = 0) -> dict:
    return {"epoch": 3, "global_step": step, "pytorch-lightning_version": "2.1.0", "loops": {}, "callbacks": {},
            "optimizer_states": [], "lr_schedulers": [], "state_dict": state_dict}


def test_golden_key_lists_agree():
    """The epipolar transformer's keys (epipolar_state_dict_keys.json) sit inside the encoder's under their name."""
    enc = {k for k, _ in json.loads((GOLDEN / "backbone_keys.json").read_text())["EncoderEpipolar"]}
    epi = json.loads((GOLDEN / "epipolar_state_dict_keys.json").read_text())["v2"]["state_dict"]
    assert {f"epipolar_transformer.{k}" for k, _ in epi} <= enc


def test_checkpoint_loads_strictly(tmp_path, encoder):
    from pixelsplat_b200.evaluation import load_checkpoint
    sd = _reference_state_dict()
    torch.save(_lightning({f"encoder.{k}": v for k, v in sd.items()}, 1234), tmp_path / "m.ckpt")
    assert load_checkpoint(tmp_path / "m.ckpt", encoder) == 1234
    for k, v in encoder.state_dict().items():
        assert torch.equal(v, sd[k]), k


@pytest.mark.parametrize("change", ["missing", "extra", "decoder", "no_state_dict"])
def test_checkpoint_rejects_other_keys(tmp_path, encoder, change):
    from pixelsplat_b200.evaluation import load_checkpoint
    sd = {f"encoder.{k}": v for k, v in _reference_state_dict().items()}
    if change == "missing":
        sd.pop("encoder.backbone.dino.cls_token")
    elif change == "extra":
        sd["encoder.to_opacity.weight"] = torch.zeros(1)
    elif change == "decoder":
        sd["decoder.background_color"] = torch.zeros(3)
    ckpt = _lightning(sd) if change != "no_state_dict" else sd
    torch.save(ckpt, tmp_path / "m.ckpt")
    with pytest.raises((RuntimeError, ValueError)) as e:
        load_checkpoint(tmp_path / "m.ckpt", encoder)
    want = {"missing": "Missing key", "extra": "Unexpected key", "decoder": "outside 'encoder.",
            "no_state_dict": "not a Lightning checkpoint"}[change]
    assert want in str(e.value)


@dataclass
class _Pickled:
    value: int


def test_checkpoint_is_read_weights_only(tmp_path, encoder):
    """A checkpoint that needs arbitrary unpickling is refused, not executed."""
    from pixelsplat_b200.evaluation import load_checkpoint
    ckpt = _lightning({f"encoder.{k}": v for k, v in _reference_state_dict().items()})
    ckpt["hyper_parameters"] = _Pickled(3)
    torch.save(ckpt, tmp_path / "m.ckpt")
    with pytest.raises(pickle.UnpicklingError):
        load_checkpoint(tmp_path / "m.ckpt", encoder)


# ---- the frame pass's C ABI: rejections happen before anything is enqueued

P = 256   # never dereferenced


def _desc(**kw):
    from pixelsplat_b200 import _lib
    d = dict(mode=_lib.PS_EVAL_RENDER, n_images=4, height=16, width=24, render=P, frame_in=0, target=P,
             frame_out=P, planes=P, sse=P)
    d.update(kw)
    return _lib.EvalDesc(*d.values())


def _call(desc, ws=P, ws_bytes=1 << 20):
    from pixelsplat_b200 import _lib
    return _lib.lib.ps_eval_images(None if desc is None else ctypes.byref(desc), ws, ws_bytes, None)


def test_abi_accepts_the_template_workspace_query():
    from pixelsplat_b200 import _lib
    from pixelsplat_b200.evaluation.frames import workspace_bytes
    assert workspace_bytes(4, 16, 24) == 256                      # one 2048-pixel tile per image, rounded to 256
    assert workspace_bytes(32, 256, 256) == 32 * 32 * 8
    for args in ((0, 16, 24), (33, 16, 24), (1, 0, 24), (1, 16, -1), (32, 20000, 20000)):
        out = ctypes.c_size_t()
        assert _lib.lib.ps_eval_images_workspace_bytes(*args, ctypes.byref(out)) == 1
    assert _lib.lib.ps_eval_images_workspace_bytes(1, 16, 24, None) == 1


@pytest.mark.parametrize("bad", [
    dict(mode=2), dict(mode=-1), dict(n_images=0), dict(n_images=33), dict(height=0), dict(width=-3),
    dict(height=20000, width=20000), dict(render=0), dict(frame_in=P), dict(mode=1), dict(mode=1, render=0, frame_in=P),
    dict(frame_out=0, planes=0, sse=0, target=0), dict(target=0), dict(sse=0), "null_desc", "null_workspace",
    "short_workspace"], ids=lambda b: b if isinstance(b, str) else "-".join(f"{k}={v}" for k, v in b.items()))
def test_abi_rejects_bad_descriptors(bad):
    from pixelsplat_b200 import _lib
    before = _lib.lib.ps_launch_count()
    if bad == "null_desc":
        rc = _call(None)
    elif bad == "null_workspace":
        rc = _call(_desc(), ws=0)
    elif bad == "short_workspace":
        rc = _call(_desc(), ws_bytes=255)
    else:
        rc = _call(_desc(**bad))
    assert rc == 1 and _lib.lib.ps_launch_count() == before
    assert b"ps_eval_images" in _lib.lib.ps_last_error()


# ---- the metric computer: skipping and aggregation

def _write_frames(root: Path, scene: str, indices) -> None:
    for i in indices:
        p = root / scene / "color" / f"{i:0>6}.png"
        p.parent.mkdir(parents=True, exist_ok=True)
        Image.fromarray(np.zeros((4, 4, 3), np.uint8)).save(p)


def test_scene_skipping(tmp_path):
    from pixelsplat_b200.evaluation import Method, scene_frame_paths
    a, b = tmp_path / "a", tmp_path / "b"
    methods = [Method("A", "a", a), Method("B", "b", b)]
    _write_frames(a, "s1", [3, 12])
    _write_frames(b, "s1", [3, 12])
    got = scene_frame_paths(methods, "s1", torch.tensor([3, 12]))
    assert got == {"a": [a / "s1/color/000003.png", a / "s1/color/000012.png"],
                   "b": [b / "s1/color/000003.png", b / "s1/color/000012.png"]}
    _write_frames(a, "s2", [1])                  # no directory for method b
    assert scene_frame_paths(methods, "s2", [1]) is None
    _write_frames(a, "s3", [1, 2])
    _write_frames(b, "s3", [1])                  # a frame is missing
    assert scene_frame_paths(methods, "s3", [1, 2]) is None
    assert scene_frame_paths(methods, "s4", [1]) is None


def test_aggregation_and_key_names():
    from pixelsplat_b200.evaluation import Method, mean_over_scenes, preview_table
    from pixelsplat_b200.evaluation.metric_computer import scene_metric_keys
    methods = [Method("Ours", "ours", Path("x")), Method("Truth", "gt", Path("y"))]
    assert scene_metric_keys(methods) == ["lpips_ours", "ssim_ours", "psnr_ours", "lpips_gt", "ssim_gt", "psnr_gt"]
    scenes = [{"psnr_ours": 20.0, "lpips_ours": 0.25, "ssim_ours": 0.5, "psnr_gt": float("inf"), "lpips_gt": 0.0,
               "ssim_gt": 1.0},
              {"psnr_ours": 30.0, "lpips_ours": 0.75, "ssim_ours": 1.0, "psnr_gt": float("inf"), "lpips_gt": 0.0,
               "ssim_gt": 1.0}]
    mean = mean_over_scenes(scenes)
    assert mean == {"psnr_ours": 25.0, "lpips_ours": 0.5, "ssim_ours": 0.75, "psnr_gt": float("inf"),
                    "lpips_gt": 0.0, "ssim_gt": 1.0}
    assert mean_over_scenes([]) == {}
    table = preview_table(mean, methods).splitlines()
    assert table[0].split() == ["Method", "PSNR", "(dB)", "LPIPS", "SSIM"]
    assert table[2].split() == ["ours", "25.000", "0.500", "0.750"] and table[3].split() == ["gt", "inf", "0.000",
                                                                                             "1.000"]


def test_per_scene_mean_is_the_mean_over_views():
    """A scene's number is the mean of its per-view values (the reference's .mean() per scene), and the result is
    the mean over scenes of those, not over all views."""
    from pixelsplat_b200.evaluation import mean_over_scenes
    per_view = [torch.tensor([10.0, 20.0, 30.0]), torch.tensor([40.0])]
    scenes = [{"psnr": float(v.mean())} for v in per_view]
    assert mean_over_scenes(scenes) == {"psnr": 30.0}


def test_presets_build_the_reference_configuration():
    from pixelsplat_b200.evaluation import presets
    assert presets.encoder_cfg("re10k") == presets.encoder_cfg("acid")
    cfg = presets.dataset_cfg("/data", "/index.json")
    assert cfg.image_shape == [256, 256] and cfg.view_sampler.num_context_views == 2
    with pytest.raises(ValueError, match="unknown preset"):
        presets.encoder_cfg("dtu")


def test_cli_parses_methods(monkeypatch):
    from pixelsplat_b200.evaluation import __main__ as cli
    with pytest.raises(SystemExit):
        cli.main(["compute-metrics", "--dataset-root", "d", "--index", "i", "--method", "no-colons"])
    with pytest.raises(SystemExit):
        cli.main(["--help"])
