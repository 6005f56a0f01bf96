"""CPU tests of the ablation and three-view presets against the reference's configuration files and modules
(fixtures of oracle/make_presets_golden.py): the composed configurations, the encoders' state dicts, checkpoint
compatibility, both command lines, and the three-view samplers on re10k_tiny."""
import dataclasses
import json
from dataclasses import replace
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import resample_oracle as ro
from oracle.make_presets_golden import ALL_PRESETS, NEW_PRESETS, TINY_SAMPLER_3, keys_crc32
from pixelsplat_b200.data import ViewSamplerBoundedCfg
from pixelsplat_b200.data.crop_shim import scaled_shape
from pixelsplat_b200.evaluation import presets as ev
from pixelsplat_b200.training import presets as tp
from tests import dataset_golden as dg

GOLDEN = Path(__file__).resolve().parent / "golden"
CONFIGS = json.loads((GOLDEN / "presets_v1.json").read_text())
KEYS = json.loads((GOLDEN / "presets_state_dict_keys.json").read_text())


def test_every_preset_is_named_in_both_commands():
    assert tuple(CONFIGS) == tuple(sorted(ALL_PRESETS))
    assert ev.PRESETS == tp.PRESETS == ALL_PRESETS and tuple(tp.TRAIN_PRESETS) == ALL_PRESETS


@pytest.mark.parametrize("name", ALL_PRESETS)
def test_preset_equals_the_reference_configuration(name):
    want = CONFIGS[name]
    preset = tp.train_preset(name)
    got = dataclasses.asdict(ev.encoder_cfg(preset.model))
    assert got.pop("visualizer") is None
    assert got == want["encoder"]
    assert dataclasses.asdict(preset.view_sampler) == want["view_sampler"]
    assert (preset.batch_size, preset.max_steps, list(preset.losses)) == \
        (want["batch_size"], want["max_steps"], want["losses"])
    views = want["view_sampler"]["num_context_views"]
    assert ev.num_context_views(preset.model) == views
    assert tp.dataset_cfg(preset, "/data").view_sampler.num_context_views == views
    assert ev.dataset_cfg("/data", "/index.json", preset=preset.model).view_sampler.num_context_views == views


def test_existing_presets_are_unchanged():
    """The values of the three presets that existed before the ablations, written out."""
    from pixelsplat_b200.encoder import EpipolarTransformerCfg, GaussianAdapterCfg, ImageSelfAttentionCfg
    from pixelsplat_b200.encoder.backbone import BackboneDinoCfg
    from pixelsplat_b200.encoder.encoder_epipolar import EncoderEpipolarCfg, OpacityMappingCfg
    re10k = EncoderEpipolarCfg(
        name="epipolar", d_feature=128, num_monocular_samples=32, num_surfaces=1, predict_opacity=False,
        backbone=BackboneDinoCfg("dino", "dino_vitb8", 512), visualizer=None, near_disparity=3.0,
        gaussian_adapter=GaussianAdapterCfg(0.5, 15.0, 4), apply_bounds_shim=True,
        epipolar_transformer=EpipolarTransformerCfg(ImageSelfAttentionCfg(4, 10, 2, 4, 128, 128, 256),
                                                    10, 2, 4, 32, 128, 256, 4),
        opacity_mapping=OpacityMappingCfg(0.0, 0.0, 1), gaussians_per_pixel=3, use_epipolar_transformer=True,
        use_transmittance=False)
    for name in ("re10k", "acid", "re10k_depth_loss"):
        assert ev.encoder_cfg(name) == re10k and ev.num_context_views(name) == 2
    sampler = ViewSamplerBoundedCfg("bounded", 2, 4, 45, 45, 0, 150_000, 25, 25)
    base = tp.TrainPreset("re10k", 7, 16, 300_001, 5000, 1.5e-4, 2000, 0.5, ("mse", "lpips"), 1.0, 0.05, 150_000,
                          0.25, None, False, None, sampler)
    assert tp.train_preset("re10k") == base
    assert tp.train_preset("acid") == replace(base, model="acid")
    assert tp.train_preset("re10k_depth_loss") == replace(base, max_steps=350_001, losses=("mse", "lpips", "depth"),
                                                          depth_sigma_image=12.0, depth_use_second_derivative=True,
                                                          depth_mode="depth")
    assert ev.dataset_cfg("/data", "/index.json") == ev.dataset_cfg("/data", "/index.json", preset="re10k")


@pytest.fixture(scope="module")
def encoders():
    """One randomly initialised encoder per preset that builds a distinct model, built on demand."""
    made = {}

    def get(name):
        if name not in made:
            torch.manual_seed(0)
            made[name] = ev.build_model(name, ev.dataset_cfg("/data", "/index.json", preset=name))[0]
        return made[name]

    yield get
    made.clear()


@pytest.mark.parametrize("name", NEW_PRESETS)
def test_encoder_has_the_reference_state_dict(name, encoders):
    """The same (name, shape) entries as the reference's EncoderEpipolar (the order of registration differs, which
    load_state_dict does not mind); the backbone's entries in the reference's order."""
    entries = [[k, list(v.shape)] for k, v in encoders(name).state_dict().items()]
    assert sorted(e for e in entries if not e[0].startswith("backbone.")) == sorted(KEYS[name]["entries"])
    assert keys_crc32([e for e in entries if e[0].startswith("backbone.")]) == KEYS[name]["backbone_crc32"]


def test_every_preset_has_the_re10k_backbone():
    ref = [e for e in json.loads((GOLDEN / "backbone_keys.json").read_text())["EncoderEpipolar"]
           if e[0].startswith("backbone.")]
    assert {KEYS[name]["backbone_crc32"] for name in NEW_PRESETS} == {keys_crc32(ref)}


def _save(path, encoder):
    torch.save({"epoch": 0, "global_step": 5, "state_dict": {f"encoder.{k}": v for k, v in
                                                              encoder.state_dict().items()}}, path)


@pytest.mark.parametrize("name", NEW_PRESETS)
def test_checkpoint_of_another_preset_is_rejected_with_a_hint(name, encoders, tmp_path):
    from pixelsplat_b200.evaluation import load_checkpoint
    from pixelsplat_b200.evaluation.__main__ import load_preset_checkpoint
    _save(tmp_path / "own.ckpt", encoders(name))
    _save(tmp_path / "re10k.ckpt", encoders("re10k"))
    assert load_preset_checkpoint(tmp_path / "own.ckpt", encoders(name), name) == 5
    for path, into, preset in ((tmp_path / "own.ckpt", encoders("re10k"), "re10k"),
                               (tmp_path / "re10k.ckpt", encoders(name), name)):
        with pytest.raises(RuntimeError):
            load_checkpoint(path, into)
        with pytest.raises(SystemExit, match="--preset") as info:
            load_preset_checkpoint(path, into, preset)
        assert isinstance(info.value.__cause__, RuntimeError)


def test_unknown_preset_lists_every_name():
    for call in (ev.encoder_cfg, ev.num_context_views, tp.train_preset,
                 lambda n: ev.dataset_cfg("/data", "/index.json", preset=n)):
        with pytest.raises(ValueError) as info:
            call("re10k_4_view")
        assert all(repr(name) in str(info.value) for name in ALL_PRESETS)


@pytest.mark.parametrize("name", NEW_PRESETS + ("re10k_depth_loss",))
def test_both_command_lines_accept_the_preset(name):
    from pixelsplat_b200.evaluation.__main__ import parse_evaluate
    from pixelsplat_b200.training.__main__ import parse
    assert parse(["--dataset-root", "d", "--preset", name, "--output", "o"]).preset == name
    assert parse_evaluate(["--dataset-root", "d", "--index", "i", "--checkpoint", "c", "--preset", name]).preset == name


def test_command_lines_reject_an_unknown_preset(capsys):
    from pixelsplat_b200.evaluation.__main__ import parse_evaluate
    from pixelsplat_b200.training.__main__ import parse
    for call in (lambda: parse(["--dataset-root", "d", "--preset", "dtu", "--output", "o"]),
                 lambda: parse_evaluate(["--dataset-root", "d", "--index", "i", "--checkpoint", "c", "--preset",
                                         "dtu"])):
        with pytest.raises(SystemExit):
            call()
        err = capsys.readouterr().err
        assert all(name in err for name in ALL_PRESETS)


def test_batch_size_help_names_the_preset():
    import contextlib
    import io

    from pixelsplat_b200.training.__main__ import parse
    out = io.StringIO()
    with contextlib.redirect_stdout(out), pytest.raises(SystemExit):
        parse(["--help"])
    text = " ".join(out.getvalue().split())
    assert "the preset's batch size" in text and "preset's 7" not in text


def test_view_count_mismatch_raises():
    with pytest.raises(ValueError, match="3 context views"):
        ev.build_model("re10k_3_view", ev.dataset_cfg("/data", "/index.json"))
    with pytest.raises(ValueError, match="2 context views"):
        ev.build_model("re10k_ablation_no_depth_encoding",
                       ev.dataset_cfg("/data", "/index.json", preset="re10k_3_view"))
    with pytest.raises(ValueError, match="context views"):
        ev.build_model("re10k", tp.dataset_cfg(tp.train_preset("re10k_3_view"), "/data"))


# ---- the three-view samplers on re10k_tiny


def _expected(stage: str) -> list[dict]:
    g = dict(np.load(GOLDEN / "dataset_re10k_3view_v1.npz"))
    out = []
    for i in range(int(g[f"{stage}/count"])):
        ex = {"scene": str(g[f"{stage}/scene"][i]), "flip": bool(g[f"{stage}/flip"][i])}
        for v in ("context", "target"):
            ex[v] = {k: g[f"{stage}/{i}/{v}/{k}"] for k in ("extrinsics", "intrinsics", "near", "far", "index",
                                                         "image_sha256", "image_sub")}
        out.append(ex)
    return out, int(g["train_seed"])


def _dataset(stage: str):
    if stage == "test":
        cfg = ev.dataset_cfg(dg.DATA, dg.DATA / "evaluation_index.json", dg.SHAPES["test"], preset="re10k_3_view")
        return ev.make_test_dataset(cfg)
    preset = replace(tp.train_preset("re10k_3_view"), view_sampler=ViewSamplerBoundedCfg(*TINY_SAMPLER_3))
    return tp.make_train_dataset(tp.dataset_cfg(preset, dg.DATA, image_shape=dg.SHAPES["train"]), None)


@pytest.mark.parametrize("stage", ["test", "train"])
def test_three_view_samplers_match_the_reference(stage):
    want, train_seed = _expected(stage)
    torch.manual_seed(train_seed if stage == "train" else 0)
    got = list(_dataset(stage))
    assert [e["scene"] for e in got] == [e["scene"] for e in want] and want
    assert [bool(e["flip"]) for e in got] == [e["flip"] for e in want]
    h_out, w_out = dg.SHAPES[stage]
    for g, w in zip(got, want):
        assert len(g["context"]["index"]) == 3
        if stage == "test":
            left, mid, right = g["context"]["index"].tolist()
            assert mid == (left + right) // 2
        for v in ("context", "target"):
            gv, wv = g[v], w[v]
            for k in ("index", "extrinsics", "near", "far"):
                assert np.array_equal(gv[k].numpy(), wv[k]), (g["scene"], v, k)
            h_s, w_s = scaled_shape(360, 640, (h_out, w_out))
            K = gv["intrinsics"].clone()
            K[..., 0, 0] *= w_s / w_out
            K[..., 1, 1] *= h_s / h_out
            assert np.array_equal(K.numpy(), wv["intrinsics"])
            crop = ((h_s - h_out) // 2, (w_s - w_out) // 2, h_out, w_out)
            out = np.stack([ro.resample_and_crop(img, (h_s, w_s), crop, bool(g["flip"])).transpose(2, 0, 1)
                            for img in gv["image"].numpy()])
            dg.assert_images_equal(out, wv, (g["scene"], v))
