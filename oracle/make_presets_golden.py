"""Generates the fixtures of the ablation and three-view presets under tests/golden/ from the REFERENCE at
/root/reference (read only while this runs).  Authoring container only:

    python oracle/make_presets_golden.py

TEST INFRASTRUCTURE.  Four files:

presets_v1.json
    For each preset name, the reference's composed configuration: every EncoderEpipolarCfg field (nested configs as
    dicts), the training view sampler's fields, the batch size, max_steps and the loss list.  Hydra is not available
    offline, so its composition is written out here (`compose`): config/main.yaml's defaults list (dataset re10k
    with view_sampler/bounded.yaml, the dataset-specific bounded_re10k.yaml over it, model/encoder epipolar.yaml,
    loss [mse]) with the experiment's `override` entries applied to it (backbone dino, the loss list), then
    main.yaml's own keys, then the rest of the experiment file, last, as Hydra composes `+experiment=` after
    main.yaml.  Mappings merge key by key; a scalar or a list replaces what was there.

presets_state_dict_keys.json
    For each new preset, (name, shape) of every entry of the reference EncoderEpipolar's state dict outside
    `backbone.`, built with the preset's view count set through set_cfg as oracle/epipolar_ref.py does, and
    `backbone_crc32`: the crc32 of the JSON list of its `backbone.` entries (`keys_crc32`), which equals that of the
    `backbone.` entries of backbone_keys.json's EncoderEpipolar list (checked here).

presets_encoder_v1.npz
    The reference's whole EncoderEpipolar of each new preset, with seeded_state_dict weights (seed 3), on seeded
    64 x 64 images and golden_util's "generic" camera rig, 2 context views (3 for re10k_3_view), in float64 and in
    float32.  torch.hub.load is stubbed as in make_backbone_golden.py, and the adapter's rotate_sh is bound to the
    restated e3nn of oracle/wigner_e3nn.py as in make_adapter_golden.py.  Per case `<preset>/<case>/`: every
    STRIDE-th Gaussian of means, covariances, harmonics and opacities, and the first PARAM_SLICE entries of the
    gradients of sum_k sum(w_k * output_k) (w_k = loss_weights of "<preset>/<case>/<k>") with respect to GRAD_PARAMS
    that exist.  Cases: `det` (deterministic=True); for no_probabilistic_sampling also `prob` (deterministic=False,
    torch.manual_seed(0); one bucket, so the draw cannot change the result: checked here with a second seed, up to
    float64 rounding, as two CPU runs of the encoder agree); for
    re10k_3_view `det_identity` and `det_swapped`, with torch.randperm replaced by the fixed permutation [0, 1] or
    [1, 0] of the view embeddings.  The float64 values are stored as float32 and of the float32 run only
    `<key>_f32_err`, its relative max-norm error against float64, as in the other fixtures.  A rerun reproduces
    every stored array; the three-view `_f32_err` values move by up to about 1 % of themselves, because the
    reference's float32 CPU run is not bit-reproducible.

dataset_re10k_3view_v1.npz
    The reference's DatasetRE10k on re10k_tiny with three context views, seeded as make_dataset_golden.py does:
    stage "train" with the bounded sampler at tiny gaps (TINY_SAMPLER_3, 256 x 256, augmentation on) and stage
    "test" with the evaluation index (180 x 320), in make_dataset_golden.record's layout.
"""
from __future__ import annotations

import copy
import json
import sys
import zlib
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
OUT = ROOT / "tests" / "golden"
REFERENCE = Path("/root/reference")

ALL_PRESETS = ("re10k", "acid", "re10k_depth_loss", "re10k_ablation_no_epipolar_transformer",
               "re10k_ablation_no_probabilistic_sampling", "re10k_ablation_no_depth_encoding", "re10k_3_view")
NEW_PRESETS = ALL_PRESETS[3:]
WEIGHT_SEED = 3
IMAGE_SEED = 4
IMAGE_SIZE = 64
STRIDE = 193                  # every 193rd Gaussian: the subsample walks across views, pixels and samples
PARAM_SLICE = 1024
GRAD_PARAMS = ("backbone_projection.1.weight", "high_resolution_skip.0.weight", "depth_predictor.projection.1.weight",
               "to_gaussians.1.weight", "epipolar_transformer.depth_encoding.1.weight",
               "epipolar_transformer.view_embeddings.weight")
OUTPUTS = ("means", "covariances", "harmonics", "opacities")
PERMUTATIONS = {"identity": (0, 1), "swapped": (1, 0)}
# the bounded sampler of tests/test_training_gpu.py's TINY_SAMPLER with three context views
TINY_SAMPLER_3 = ("bounded", 3, 4, 2, 6, 0, 0, 2, 6)


def num_views(preset: str) -> int:
    return 3 if preset == "re10k_3_view" else 2


def cases(preset: str) -> tuple[str, ...]:
    if preset == "re10k_3_view":
        return tuple(f"det_{p}" for p in PERMUTATIONS)
    if preset == "re10k_ablation_no_probabilistic_sampling":
        return ("det", "prob")
    return ("det",)


def keys_crc32(entries: list) -> int:
    """crc32 of a JSON list of [name, shape] state-dict entries."""
    return zlib.crc32(json.dumps([[k, list(s)] for k, s in entries]).encode())


# ---- the configuration, composed from the reference's yaml files


def _merge(a, b):
    if isinstance(a, dict) and isinstance(b, dict):
        out = dict(a)
        for k, v in b.items():
            out[k] = _merge(a[k], v) if k in a else copy.deepcopy(v)
        return out
    return copy.deepcopy(b)


def _yaml(rel: str) -> dict:
    import yaml
    doc = yaml.safe_load((REFERENCE / "config" / rel).read_text())
    doc.pop("defaults", None)
    return doc


def compose(preset: str) -> dict:
    """The parts of the composed config the presets set (see the module docstring for the precedence)."""
    import yaml
    exp_doc = yaml.safe_load((REFERENCE / "config" / "experiment" / f"{preset}.yaml").read_text())
    overrides = {k: v for d in exp_doc.pop("defaults") for k, v in d.items()}
    # main.yaml's defaults list, with the experiment's overrides of its groups (dataset and encoder stay as main.yaml
    # names them; the experiments override them with the same values)
    assert overrides["override /dataset"] == "re10k" and overrides["override /model/encoder"] == "epipolar"
    dataset = _merge(_yaml("dataset/re10k.yaml"), {"view_sampler": _yaml("dataset/view_sampler/bounded.yaml")})
    cfg = _merge({"dataset": dataset}, _yaml("dataset/view_sampler_dataset_specific_config/bounded_re10k.yaml"))
    encoder = _yaml("model/encoder/epipolar.yaml")
    encoder["backbone"] = _yaml(f"model/encoder/backbone/{overrides['override /model/encoder/backbone']}.yaml")
    cfg = _merge(cfg, {"model": {"encoder": encoder}})
    losses = list(overrides.get("override /loss", ["mse"]))
    cfg = _merge(cfg, _yaml("main.yaml"))          # main.yaml's own keys after its defaults
    cfg = _merge(cfg, exp_doc)                     # the experiment last
    enc = cfg["model"]["encoder"]
    enc.pop("visualizer")
    return {"encoder": enc, "view_sampler": cfg["dataset"]["view_sampler"],
            "batch_size": cfg["data_loader"]["train"]["batch_size"], "max_steps": cfg["trainer"]["max_steps"],
            "losses": losses}


# ---- the reference encoder


def _load_reference(views: int):
    from oracle import epipolar_ref, make_backbone_golden, wigner_e3nn
    make_backbone_golden._load_reference()
    epipolar_ref.load(views)                        # set_cfg: the view count EpipolarTransformer reads
    from src.model.encoder import encoder_epipolar
    from src.model.encoder.backbone.backbone_dino import BackboneDinoCfg
    from src.model.encoder.common import gaussian_adapter
    from src.model.encoder.common.gaussian_adapter import GaussianAdapterCfg
    from src.model.encoder.epipolar.epipolar_transformer import EpipolarTransformerCfg
    from src.model.encoder.epipolar.image_self_attention import ImageSelfAttentionCfg
    gaussian_adapter.rotate_sh = wigner_e3nn.rotate_sh_reference
    if not hasattr(gaussian_adapter.GaussianAdapter, "_float32_pixel_size"):
        # the reference hard-codes a float32 pixel_size (gaussian_adapter.py:67); cast it as make_adapter_golden.py
        # does (1/w and 1/h are formed in float32 exactly as upstream)
        orig = gaussian_adapter.GaussianAdapter.get_scale_multiplier
        gaussian_adapter.GaussianAdapter.get_scale_multiplier = \
            lambda self, K, ps, *a: orig(self, K, ps.to(K.dtype), *a)
        gaussian_adapter.GaussianAdapter._float32_pixel_size = orig
    return encoder_epipolar, BackboneDinoCfg, GaussianAdapterCfg, EpipolarTransformerCfg, ImageSelfAttentionCfg


def reference_encoder(preset: str):
    encoder_epipolar, BackboneDinoCfg, GaussianAdapterCfg, EpipolarTransformerCfg, ImageSelfAttentionCfg = \
        _load_reference(num_views(preset))
    e = compose(preset)["encoder"]
    et = e["epipolar_transformer"]
    sa = ImageSelfAttentionCfg(**et.pop("self_attention"))
    cfg = encoder_epipolar.EncoderEpipolarCfg(
        **{k: v for k, v in e.items() if k not in ("backbone", "gaussian_adapter", "epipolar_transformer",
                                                    "opacity_mapping")},
        visualizer=None, backbone=BackboneDinoCfg(**e["backbone"]),
        gaussian_adapter=GaussianAdapterCfg(**e["gaussian_adapter"]),
        epipolar_transformer=EpipolarTransformerCfg(self_attention=sa, **et),
        opacity_mapping=encoder_epipolar.OpacityMappingCfg(**e["opacity_mapping"]))
    return encoder_epipolar.EncoderEpipolar(cfg)


def inputs(views: int, dtype=torch.float64) -> dict:
    """The context of the encoder fixtures: seeded images and golden_util's generic rig (batch 1)."""
    from oracle.make_backbone_golden import images
    from tests import golden_util as gu
    ext, K, near, far = gu.camera_rig(1, views, "generic")
    image = images((1, views, 3, IMAGE_SIZE, IMAGE_SIZE), IMAGE_SEED)
    return {k: t.to(dtype) for k, t in dict(image=image, extrinsics=ext, intrinsics=K, near=near, far=far).items()}


def output_arrays(gaussians) -> dict:
    return {k: getattr(gaussians, k)[:, ::STRIDE] for k in OUTPUTS}


def weighted_sum(outputs: dict, prefix: str) -> torch.Tensor:
    from oracle.make_backbone_golden import loss_weights
    return sum((y.double() * loss_weights(y.shape, f"{prefix}{k}").to(y.device)).sum() for k, y in outputs.items())


class fixed_randperm:
    """Replaces torch.randperm (the view embeddings' shuffle) by a fixed permutation while active."""

    def __init__(self, perm):
        self.perm = perm

    def __enter__(self):
        self.original = torch.randperm

        def randperm(n, *args, device=None, **kwargs):
            assert n == len(self.perm), (n, self.perm)
            return torch.tensor(self.perm, dtype=torch.int64, device=device)

        torch.randperm = randperm

    def __exit__(self, *exc):
        torch.randperm = self.original


def run_case(encoder, preset: str, case: str, dtype, seed: int = 0):
    """(outputs, gradients) of one case as float64 numpy arrays."""
    import contextlib
    context = inputs(num_views(preset), dtype)
    perm = case.split("_", 1)[1] if case.startswith("det_") else None
    encoder.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    with fixed_randperm(PERMUTATIONS[perm]) if perm else contextlib.nullcontext():
        g = encoder(context, global_step=0, deterministic=case.startswith("det"))
    out = output_arrays(g)
    weighted_sum(out, f"{preset}/{case}/").backward()
    params = dict(encoder.named_parameters())
    grads = {f"d_{k}": params[k].grad.detach().reshape(-1)[:PARAM_SLICE] for k in GRAD_PARAMS if k in params}
    return ({k: v.detach().double().numpy() for k, v in out.items()},
            {k: v.double().numpy() for k, v in grads.items()})


def encoder_fixture(keys_out: dict) -> dict:
    from oracle.make_backbone_golden import rel_err, seeded_state_dict
    backbone_ref = [e for e in json.loads((OUT / "backbone_keys.json").read_text())["EncoderEpipolar"]
                    if e[0].startswith("backbone.")]
    out = {}
    for preset in NEW_PRESETS:
        res = {}
        for dtype, tag in ((torch.float64, "f64"), (torch.float32, "f32")):
            torch.set_default_dtype(dtype)      # the reference builds its grids in the default dtype
            enc = reference_encoder(preset)
            enc.load_state_dict(seeded_state_dict(enc, WEIGHT_SEED))
            enc = enc.to(dtype).eval()
            enc.gaussian_adapter.sh_mask = enc.gaussian_adapter.sh_mask.to(dtype)
            if tag == "f64":
                entries = [[k, list(v.shape)] for k, v in enc.state_dict().items()]
                backbone = [e for e in entries if e[0].startswith("backbone.")]
                assert keys_crc32(backbone) == keys_crc32(backbone_ref), f"{preset}: not the re10k backbone"
                keys_out[preset] = {"entries": [e for e in entries if not e[0].startswith("backbone.")],
                                    "backbone_crc32": keys_crc32(backbone)}
            for case in cases(preset):
                o, g = run_case(enc, preset, case, dtype)
                res[(tag, case)] = {**o, **g}
                if case == "prob" and tag == "f64":
                    o2, _ = run_case(enc, preset, case, dtype, seed=1)
                    diff = {k: float(np.abs(o[k] - o2[k]).max() / np.abs(o[k]).max()) for k in o}
                    assert max(diff.values()) < 1e-12, f"one bucket: the draw changed the result {diff}"
            torch.set_default_dtype(torch.float32)
        for case in cases(preset):
            for k, ref in res[("f64", case)].items():
                key = f"{preset}/{case}/{k}"
                out[key] = ref.astype(np.float32)
                out[key + "_f32_err"] = np.array(rel_err(res[("f32", case)][k], ref))
    return out


# ---- the three-view dataset


def dataset_fixture() -> dict:
    from oracle import make_dataset_golden as mdg
    ds_mod, vs_mod = mdg.load_reference()
    from omegaconf import DictConfig
    from src.global_cfg import set_cfg
    set_cfg(DictConfig({"dataset": {"view_sampler": {"num_context_views": 3}}}))
    train_seed = int(np.load(OUT / "dataset_re10k_v1.npz")["train_seed"])
    fixture = {"train_seed": np.array(train_seed)}
    for stage, seed in (("test", 0), ("train", train_seed)):
        if stage == "test":
            vs = vs_mod.ViewSamplerEvaluationCfg("evaluation", mdg.DATA / "evaluation_index.json", 3)
            shape = mdg.TEST_SHAPE
        else:
            vs = vs_mod.ViewSamplerBoundedCfg(*TINY_SAMPLER_3)
            shape = mdg.TRAIN_SHAPE
        cfg = ds_mod.DatasetRE10kCfg(image_shape=list(shape), background_color=[0.0, 0.0, 0.0],
                                     cameras_are_circular=False, overfit_to_scene=None, view_sampler=vs,
                                     name="re10k", roots=[mdg.DATA], baseline_epsilon=1e-3, max_fov=100.0,
                                     make_baseline_1=True, augment=True)
        flips = []
        original = ds_mod.apply_augmentation_shim

        def recording(example, generator=None):
            result = original(example, generator)
            flips.append(result is not example)
            return result

        ds_mod.apply_augmentation_shim = recording
        try:
            torch.manual_seed(seed)
            examples = list(ds_mod.DatasetRE10k(cfg, stage, vs_mod.get_view_sampler(vs, stage, False, False, None)))
        finally:
            ds_mod.apply_augmentation_shim = original
        if stage != "train":
            flips = [False] * len(examples)
        for ex, f in zip(examples, flips):
            ex["flip"] = f
            assert len(ex["context"]["index"]) == 3
        fixture.update(mdg.record(examples, stage))
    return fixture


def main() -> None:
    torch.set_grad_enabled(True)
    presets = {name: compose(name) for name in ALL_PRESETS}
    (OUT / "presets_v1.json").write_text(json.dumps(presets, indent=1, sort_keys=True) + "\n")
    keys = {}
    enc = encoder_fixture(keys)
    (OUT / "presets_state_dict_keys.json").write_text(json.dumps(keys, indent=0) + "\n")
    np.savez_compressed(OUT / "presets_encoder_v1.npz", **enc)
    data = dataset_fixture()
    np.savez_compressed(OUT / "dataset_re10k_3view_v1.npz", **data)
    for name in ("presets_v1.json", "presets_state_dict_keys.json", "presets_encoder_v1.npz",
                 "dataset_re10k_3view_v1.npz"):
        print(f"{name}: {(OUT / name).stat().st_size / 1e3:.0f} kB")
    print({k: float(v) for k, v in enc.items() if k.endswith("_f32_err")})


if __name__ == "__main__":
    main()
