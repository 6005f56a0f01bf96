"""Generates tests/golden/backbone_*.npz and backbone_keys.json by running the REFERENCE's BackboneResnet,
BackboneDino and EncoderEpipolar from /root/reference on the CPU (float64 and float32).  Authoring container only:

    python oracle/make_backbone_golden.py

TEST INFRASTRUCTURE.  The reference builds DINO's models through torch.hub.load, which needs the network; here
torch.hub.load is replaced by a stub returning this package's restated VisionTransformer or torchvision's resnet50
with fc = Identity (what DINO's hub entry builds).  Everything else is the reference's own code: the ResNet
projections, the align-corners upsampling and the sum, the token MLPs and their repeats, and the encoder's
composition.  So the fixtures pin that wiring, not DINO's internals (see DESIGN.md section 6).

Weights come from seeded_state_dict (below), which the tests call with the same seed: no weights are stored.
To keep the fixture small, only a subsample of each result is stored (`sub`, `sub_image`, the first PARAM_SLICE
entries of a parameter gradient, every 8th token and channel of the ViT), the float64 values as float32 (a
relative rounding of 6e-8, far below every bar), and of the reference's float32 run only its relative max-norm
error against float64 on that subsample (`<key>_f32_err`), which is what the tests' bars are built from.
"""
from __future__ import annotations

import json
import sys
import zlib
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
OUT = ROOT / "tests" / "golden"


def seeded_state_dict(module: torch.nn.Module, seed: int) -> dict:
    """Deterministic weights for `module`'s state dict: one torch.Generator per floating-point entry, in key order,
    seeded with (seed, crc32 of the key), so the values depend on the key's name only.  Matrices and kernels are
    N(0, 1 / fan_in); 1-D `weight`s (norm scales) 1 + N(0, 0.1^2); BatchNorm running variances 1 + U(0, 0.5);
    everything else N(0, 0.1^2).  Integer buffers (num_batches_tracked) are kept."""
    out = {}
    for key, v in module.state_dict().items():
        if not v.is_floating_point():
            out[key] = v.clone()
            continue
        g = torch.Generator().manual_seed(seed * 1_000_003 + zlib.crc32(key.encode()))
        if key.endswith("running_var"):
            x = 1.0 + 0.5 * torch.rand(v.shape, generator=g, dtype=torch.float64)
        elif v.dim() > 1 and not key.endswith(("cls_token", "pos_embed")):
            x = torch.randn(v.shape, generator=g, dtype=torch.float64) / np.sqrt(v[0].numel())
        elif key.endswith("weight") and v.dim() == 1:
            x = 1.0 + 0.1 * torch.randn(v.shape, generator=g, dtype=torch.float64)
        else:
            x = 0.1 * torch.randn(v.shape, generator=g, dtype=torch.float64)
        out[key] = x.to(v.dtype)
    return out


def sub(y: torch.Tensor) -> torch.Tensor:
    """The stored part of a [b, v, c, h, w] feature map: every 16th channel, every 4th row and column."""
    return y[:, :, ::16, ::4, ::4]


def sub_image(g: torch.Tensor) -> torch.Tensor:
    """The stored part of an image gradient [b, v, 3, h, w]: every 2nd row and column."""
    return g[..., ::2, ::2]


def sub_tokens(t: torch.Tensor) -> torch.Tensor:
    """The stored part of ViT tokens [n, L, c]: every 8th token and every 8th channel."""
    return t[:, ::8, ::8]


def rel_err(a: np.ndarray, b: np.ndarray) -> float:
    """Relative max-norm error of a against b."""
    return float(np.abs(a - b).max() / np.abs(b).max())


def images(shape, seed: int) -> torch.Tensor:
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def loss_weights(shape, name: str) -> torch.Tensor:
    """Fixed random weights w of the scalar loss sum(w * output) whose gradients the fixtures store."""
    return torch.randn(shape, generator=torch.Generator().manual_seed(zlib.crc32(name.encode())), dtype=torch.float64)


# the reference encoder config of config/experiment/re10k.yaml (backbone dino_vitb8, d_out 512)
RE10K = dict(d_feature=128, num_monocular_samples=32, num_surfaces=1, predict_opacity=False, near_disparity=3.0,
             apply_bounds_shim=True, gaussians_per_pixel=3, use_epipolar_transformer=True, use_transmittance=False)
PARAM_SLICES = ("dino.blocks.11.attn.qkv.weight", "dino.patch_embed.proj.weight", "local_token_mlp.2.weight",
                "resnet_backbone.projections.layer0.weight", "resnet_backbone.model.layer3.0.conv1.weight")
PARAM_SLICE = 1024


def _load_reference():
    from oracle import epipolar_ref
    from pixelsplat_b200.encoder import backbone as ours
    epipolar_ref.load(2)

    def hub_load(repo, model, *args, **kwargs):
        return ours.DINO_BUILDERS[model]()

    torch.hub.load = hub_load
    import types
    for name in ("src.model.encoder.common", "src.model.encoder.epipolar",
                 "src.model.encoder.visualization", "src.dataset.shims"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__path__ = [str(epipolar_ref.REFERENCE / name.replace(".", "/"))]
            sys.modules[name] = m
    from src.model.encoder.backbone import backbone_dino, backbone_resnet
    return backbone_dino, backbone_resnet


def main() -> None:
    backbone_dino, backbone_resnet = _load_reference()
    torch.set_grad_enabled(True)
    keys, res = {}, {"f64": {}, "f32": {}}

    def run(module, x, name, dtype):
        module = module.to(dtype).eval()
        xi = x.to(dtype).clone().requires_grad_(True)
        y = module({"image": xi})
        (y.double() * loss_weights(y.shape, name)).sum().backward()
        return sub(y.detach().double()).numpy(), sub_image(xi.grad.double()).numpy(), module

    # BackboneResnet(resnet50, 5 layers): the InstanceNorm ResNet, 2 views of 64 x 64
    cfg = backbone_resnet.BackboneResnetCfg("resnet", "resnet50", 5, False, 512)
    x = images((1, 2, 3, 64, 64), 1)
    for dtype, tag in ((torch.float64, "f64"), (torch.float32, "f32")):
        m = backbone_resnet.BackboneResnet(cfg, 3)
        m.load_state_dict(seeded_state_dict(m, 0))
        y, gx, m = run(m, x, "resnet", dtype)
        res[tag]["resnet_out"], res[tag]["resnet_d_image"] = y, gx
    keys["BackboneResnet"] = [[k, list(v.shape)] for k, v in m.state_dict().items()]

    # BackboneDino(dino_vitb8, d_out 512): 2 views of 64 x 64
    cfg = backbone_dino.BackboneDinoCfg("dino", "dino_vitb8", 512)
    for dtype, tag in ((torch.float64, "f64"), (torch.float32, "f32")):
        m = backbone_dino.BackboneDino(cfg, 3)
        m.load_state_dict(seeded_state_dict(m, 1))
        y, gx, m = run(m, x, "dino", dtype)
        res[tag]["dino_out"], res[tag]["dino_d_image"] = y, gx
        params = dict(m.named_parameters())
        for k in PARAM_SLICES:
            res[tag][f"dino_d_{k}"] = params[k].grad.detach().double().reshape(-1)[:PARAM_SLICE].numpy()
    keys["BackboneDino"] = [[k, list(v.shape)] for k, v in m.state_dict().items()]

    # the ViT alone at the re10k shape: 256 x 256, patch 8 -> L = 1 + 32 * 32 = 1025 tokens
    from pixelsplat_b200.encoder import backbone as ours
    x256 = images((1, 3, 256, 256), 2)
    for dtype, tag in ((torch.float64, "f64"), (torch.float32, "f32")):
        vit = ours.dino_vitb8()
        vit.load_state_dict(seeded_state_dict(vit, 2))
        vit = vit.to(dtype)
        tok = vit.get_intermediate_layers(x256.to(dtype))[0]
        res[tag]["vit256_tokens"] = sub_tokens(tok.detach().double()).numpy()

    # EncoderEpipolar with the re10k config: state-dict keys and shapes
    try:
        from src.model.encoder import encoder_epipolar
        from src.model.encoder.common.gaussian_adapter import GaussianAdapterCfg
        from src.model.encoder.epipolar.epipolar_transformer import EpipolarTransformerCfg
        from src.model.encoder.epipolar.image_self_attention import ImageSelfAttentionCfg
        enc_cfg = encoder_epipolar.EncoderEpipolarCfg(
            name="epipolar", backbone=cfg, visualizer=None,
            gaussian_adapter=GaussianAdapterCfg(0.5, 15.0, 4),
            epipolar_transformer=EpipolarTransformerCfg(ImageSelfAttentionCfg(4, 10, 2, 4, 128, 128, 256),
                                                        10, 2, 4, 32, 128, 256, 4),
            opacity_mapping=encoder_epipolar.OpacityMappingCfg(0.0, 0.0, 1), **RE10K)
        enc = encoder_epipolar.EncoderEpipolar(enc_cfg)
        keys["EncoderEpipolar"] = [[k, list(v.shape)] for k, v in enc.state_dict().items()]
    except ImportError as exc:
        raise SystemExit(f"reference EncoderEpipolar not importable: {exc}")

    out = {}
    for k, ref in res["f64"].items():
        out[k] = ref.astype(np.float32)
        out[k + "_f32_err"] = np.array(rel_err(res["f32"][k], ref))
    np.savez_compressed(OUT / "backbone_v1.npz", **out)
    (OUT / "backbone_keys.json").write_text(json.dumps(keys, indent=0))
    print({k: len(v) for k, v in keys.items()}, sorted(out))


if __name__ == "__main__":
    main()
