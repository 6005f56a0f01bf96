"""Image backbones of pixelSplat's encoder: the reference's `BackboneResnet`, `BackboneDino` and `get_backbone`
(src/model/encoder/backbone/{backbone_resnet,backbone_dino,__init__}.py), with the same constructor arguments,
parameter names and `[b, v, d_out, h, w]` output.

`VisionTransformer` restates DINO's vision_transformer.py (facebookresearch/dino) with DINO's parameter names, so
its released checkpoints load with strict=True.  The attention of every block runs on the flash-style sm_90a kernel
(csrc/vit_attention.cu) when the input is CUDA fp32 with 64-dim heads (ViT-S and ViT-B);
PIXELSPLAT_B200_VIT_ATTENTION=fp32 selects DINO's explicit formula instead.  The GEMMs, LayerNorms and the
ResNet-50 convolutions stay on cuBLAS / cuDNN.

Weights are never downloaded.  Without weights, modules are randomly initialised (enough to load a pixelSplat
checkpoint, which holds the backbone's weights anyway).  `pretrained=True` or `from_files(...)` reads DINO's
released `.pth` files from the torch hub checkpoint directory or from given paths.
"""
from __future__ import annotations

import functools
import math
import os
from dataclasses import dataclass
from pathlib import Path
from typing import Literal

import torch
import torch.nn.functional as F
import torchvision
from torch import Tensor, nn

from . import vit_attention as va

# DINO's released checkpoints, as torch.hub stores them under <hub dir>/checkpoints
DINO_FILES = {
    "dino_vits16": "dino_deitsmall16_pretrain.pth",
    "dino_vits8": "dino_deitsmall8_pretrain.pth",
    "dino_vitb16": "dino_vitbase16_pretrain.pth",
    "dino_vitb8": "dino_vitbase8_pretrain.pth",
    "dino_resnet50": "dino_resnet50_pretrain.pth",
}


# ---------------------------------------------------------------------------------------------------------------
# DINO's VisionTransformer (no dropout, no drop-path: the hub models are built with rate 0)


class PatchEmbed(nn.Module):
    def __init__(self, img_size: int = 224, patch_size: int = 16, in_chans: int = 3, embed_dim: int = 768) -> None:
        super().__init__()
        self.img_size, self.patch_size = img_size, patch_size
        self.num_patches = (img_size // patch_size) * (img_size // patch_size)
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)

    def forward(self, x: Tensor) -> Tensor:
        return self.proj(x).flatten(2).transpose(1, 2)


class Attention(nn.Module):
    def __init__(self, dim: int, num_heads: int, qkv_bias: bool = True) -> None:
        super().__init__()
        self.num_heads = num_heads
        head_dim = dim // num_heads
        self.scale = head_dim ** -0.5
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)

    def forward(self, x: Tensor) -> Tensor:
        B, N, C = x.shape
        H = self.num_heads
        qkv = self.qkv(x)                                            # [B, N, (3 H d)]
        if va.supported(qkv, H, C // H):
            out = va.vit_attention(qkv, H, self.scale)
        else:
            q, k, v = qkv.reshape(B, N, 3, H, C // H).permute(2, 0, 3, 1, 4)
            attn = ((q @ k.transpose(-2, -1)) * self.scale).softmax(dim=-1)
            out = (attn @ v).transpose(1, 2).reshape(B, N, C)
        return self.proj(out)


class Mlp(nn.Module):
    def __init__(self, dim: int, hidden: int) -> None:
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden, dim)

    def forward(self, x: Tensor) -> Tensor:
        return self.fc2(self.act(self.fc1(x)))


class Block(nn.Module):
    def __init__(self, dim: int, num_heads: int, mlp_ratio: float = 4.0) -> None:
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=1e-6)
        self.attn = Attention(dim, num_heads)
        self.norm2 = nn.LayerNorm(dim, eps=1e-6)
        self.mlp = Mlp(dim, int(dim * mlp_ratio))

    def forward(self, x: Tensor) -> Tensor:
        x = x + self.attn(self.norm1(x))
        return x + self.mlp(self.norm2(x))


class VisionTransformer(nn.Module):
    def __init__(self, patch_size: int = 16, embed_dim: int = 768, depth: int = 12, num_heads: int = 12,
                 mlp_ratio: float = 4.0, img_size: int = 224, in_chans: int = 3) -> None:
        super().__init__()
        self.num_features = self.embed_dim = embed_dim
        self.patch_embed = PatchEmbed(img_size, patch_size, in_chans, embed_dim)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.pos_embed = nn.Parameter(torch.zeros(1, self.patch_embed.num_patches + 1, embed_dim))
        self.blocks = nn.ModuleList([Block(embed_dim, num_heads, mlp_ratio) for _ in range(depth)])
        self.norm = nn.LayerNorm(embed_dim, eps=1e-6)
        self.head = nn.Identity()
        nn.init.trunc_normal_(self.pos_embed, std=0.02)
        nn.init.trunc_normal_(self.cls_token, std=0.02)
        self.apply(self._init_weights)

    @staticmethod
    def _init_weights(m: nn.Module) -> None:
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.zeros_(m.bias)
        elif isinstance(m, nn.LayerNorm):
            nn.init.ones_(m.weight)
            nn.init.zeros_(m.bias)

    def interpolate_pos_encoding(self, x: Tensor, w: int, h: int) -> Tensor:
        """DINO's bicubic resampling of the 224-pixel position grid, with its +0.1 offset against floating-point
        error in the scale factor; `w` is the image's height and `h` its width (DINO's names, see prepare_tokens)."""
        npatch = x.shape[1] - 1
        N = self.pos_embed.shape[1] - 1
        if npatch == N and w == h:
            return self.pos_embed
        class_pos_embed = self.pos_embed[:, 0]
        patch_pos_embed = self.pos_embed[:, 1:]
        dim = x.shape[-1]
        w0 = w // self.patch_embed.patch_size + 0.1
        h0 = h // self.patch_embed.patch_size + 0.1
        patch_pos_embed = F.interpolate(
            patch_pos_embed.reshape(1, int(math.sqrt(N)), int(math.sqrt(N)), dim).permute(0, 3, 1, 2),
            scale_factor=(w0 / math.sqrt(N), h0 / math.sqrt(N)), mode="bicubic")
        assert int(w0) == patch_pos_embed.shape[-2] and int(h0) == patch_pos_embed.shape[-1]
        patch_pos_embed = patch_pos_embed.permute(0, 2, 3, 1).view(1, -1, dim)
        return torch.cat((class_pos_embed.unsqueeze(0), patch_pos_embed), dim=1)

    def prepare_tokens(self, x: Tensor) -> Tensor:
        B, nc, w, h = x.shape                                       # DINO's names: w is the height
        x = self.patch_embed(x)
        x = torch.cat((self.cls_token.expand(B, -1, -1), x), dim=1)
        return x + self.interpolate_pos_encoding(x, w, h)

    def forward(self, x: Tensor) -> Tensor:
        x = self.prepare_tokens(x)
        for blk in self.blocks:
            x = blk(x)
        return self.norm(x)[:, 0]

    def get_intermediate_layers(self, x: Tensor, n: int = 1) -> list[Tensor]:
        """The final norm applied to the outputs of the last n blocks."""
        x = self.prepare_tokens(x)
        output = []
        for i, blk in enumerate(self.blocks):
            x = blk(x)
            if len(self.blocks) - i <= n:
                output.append(self.norm(x))
        return output


def dino_vits16() -> VisionTransformer:
    return VisionTransformer(patch_size=16, embed_dim=384, depth=12, num_heads=6)


def dino_vits8() -> VisionTransformer:
    return VisionTransformer(patch_size=8, embed_dim=384, depth=12, num_heads=6)


def dino_vitb16() -> VisionTransformer:
    return VisionTransformer(patch_size=16, embed_dim=768, depth=12, num_heads=12)


def dino_vitb8() -> VisionTransformer:
    return VisionTransformer(patch_size=8, embed_dim=768, depth=12, num_heads=12)


def dino_resnet50() -> nn.Module:
    """What DINO's hub entry builds: torchvision's resnet50 (BatchNorm) without its classifier."""
    model = torchvision.models.resnet50()
    model.fc = nn.Identity()
    return model


DINO_BUILDERS = {"dino_vits16": dino_vits16, "dino_vits8": dino_vits8, "dino_vitb16": dino_vitb16,
                 "dino_vitb8": dino_vitb8, "dino_resnet50": dino_resnet50}


# ---------------------------------------------------------------------------------------------------------------
# weights from files


def hub_checkpoint_dir() -> Path:
    return Path(torch.hub.get_dir()) / "checkpoints"


def dino_weights_path(model: str, path: str | os.PathLike | None = None) -> Path:
    """`path` if given, else DINO's released file for `model` in the torch hub checkpoint directory.  A missing file
    raises FileNotFoundError naming what it should hold; nothing is downloaded."""
    p = Path(path) if path is not None else hub_checkpoint_dir() / DINO_FILES[model]
    if not p.is_file():
        raise FileNotFoundError(
            f"{p} not found: it should hold DINO's released {model} weights ({DINO_FILES[model]}). Pass its path "
            f"or place it in {hub_checkpoint_dir()}; weights are never downloaded.")
    return p


def load_dino_weights(module: nn.Module, model: str, path: str | os.PathLike | None = None) -> None:
    state = torch.load(dino_weights_path(model, path), map_location="cpu", weights_only=True)
    if model == "dino_resnet50":
        # DINO's hub entry loads with strict=False: the checkpoint has no classifier (fc is an Identity)
        missing, unexpected = module.load_state_dict(state, strict=False)
        if missing or unexpected:
            raise RuntimeError(f"dino_resnet50 weights: missing {missing}, unexpected {unexpected}")
    else:
        module.load_state_dict(state, strict=True)


# ---------------------------------------------------------------------------------------------------------------
# the reference's backbones


@dataclass
class BackboneResnetCfg:
    name: Literal["resnet"]
    model: Literal["resnet18", "resnet34", "resnet50", "resnet101", "resnet152", "dino_resnet50"]
    num_layers: int
    use_first_pool: bool
    d_out: int


class BackboneResnet(nn.Module):
    """A torchvision ResNet with the reference's InstanceNorm2d norm layer (or DINO's ResNet-50), 1x1 projections of
    layer0 .. layer{num_layers - 1} to d_out, align-corners bilinear upsampling to the image size, and their sum."""

    def __init__(self, cfg: BackboneResnetCfg, d_in: int, pretrained: bool = False,
                 weights_path: str | os.PathLike | None = None) -> None:
        super().__init__()
        self.cfg = cfg
        assert d_in == 3
        norm_layer = functools.partial(nn.InstanceNorm2d, affine=False, track_running_stats=False)
        if cfg.model == "dino_resnet50":
            self.model = dino_resnet50()
            if pretrained or weights_path is not None:
                load_dino_weights(self.model, "dino_resnet50", weights_path)
        else:
            self.model = getattr(torchvision.models, cfg.model)(norm_layer=norm_layer)

        self.projections = nn.ModuleDict({})
        for index in range(1, cfg.num_layers):
            key = f"layer{index}"
            block = getattr(self.model, key)
            conv_index = 1
            try:
                while True:
                    d_layer_out = getattr(block[-1], f"conv{conv_index}").out_channels
                    conv_index += 1
            except AttributeError:
                pass
            self.projections[key] = nn.Conv2d(d_layer_out, cfg.d_out, 1)
        self.projections["layer0"] = nn.Conv2d(self.model.conv1.out_channels, cfg.d_out, 1)

    def forward(self, context: dict) -> Tensor:
        b, v, _, h, w = context["image"].shape
        x = context["image"].reshape(b * v, *context["image"].shape[2:])
        x = self.model.relu(self.model.bn1(self.model.conv1(x)))
        features = [self.projections["layer0"](x)]
        for index in range(1, self.cfg.num_layers):
            key = f"layer{index}"
            if index == 0 and self.cfg.use_first_pool:               # the reference's condition: never true
                x = self.model.maxpool(x)
            x = getattr(self.model, key)(x)
            features.append(self.projections[key](x))
        features = [F.interpolate(f, (h, w), mode="bilinear", align_corners=True) for f in features]
        features = torch.stack(features).sum(dim=0)
        return features.reshape(b, v, *features.shape[1:])

    @property
    def d_out(self) -> int:
        return self.cfg.d_out


@dataclass
class BackboneDinoCfg:
    name: Literal["dino"]
    model: Literal["dino_vits16", "dino_vits8", "dino_vitb16", "dino_vitb8"]
    d_out: int


class BackboneDino(nn.Module):
    """DINO's ViT and DINO's ResNet-50: the ResNet's projected pyramid plus the ViT's last-layer tokens through two
    MLPs, the CLS token broadcast over the image and each patch token repeated over its patch."""

    def __init__(self, cfg: BackboneDinoCfg, d_in: int, pretrained: bool = False) -> None:
        super().__init__()
        self.cfg = cfg
        assert d_in == 3
        self.dino = DINO_BUILDERS[cfg.model]()
        if pretrained:
            load_dino_weights(self.dino, cfg.model)
        self.resnet_backbone = BackboneResnet(BackboneResnetCfg("resnet", "dino_resnet50", 4, False, cfg.d_out),
                                              d_in, pretrained=pretrained)
        self.global_token_mlp = nn.Sequential(nn.Linear(768, 768), nn.ReLU(), nn.Linear(768, cfg.d_out))
        self.local_token_mlp = nn.Sequential(nn.Linear(768, 768), nn.ReLU(), nn.Linear(768, cfg.d_out))

    @classmethod
    def from_files(cls, cfg: BackboneDinoCfg, d_in: int = 3, vit_path: str | os.PathLike | None = None,
                   resnet_path: str | os.PathLike | None = None) -> "BackboneDino":
        """A BackboneDino with DINO's released weights read from `vit_path` / `resnet_path`, or, for a path not
        given, from the torch hub checkpoint directory under the released file name.  Never downloads."""
        vit_file = dino_weights_path(cfg.model, vit_path)
        resnet_file = dino_weights_path("dino_resnet50", resnet_path)
        module = cls(cfg, d_in)
        load_dino_weights(module.dino, cfg.model, vit_file)
        load_dino_weights(module.resnet_backbone.model, "dino_resnet50", resnet_file)
        return module

    def forward(self, context: dict) -> Tensor:
        resnet_features = self.resnet_backbone(context)
        b, v, _, h, w = context["image"].shape
        p = self.patch_size
        assert h % p == 0 and w % p == 0
        tokens = context["image"].reshape(b * v, *context["image"].shape[2:])
        tokens = self.dino.get_intermediate_layers(tokens)[0]
        global_token = self.global_token_mlp(tokens[:, 0])                         # [(b v), c]
        local_tokens = self.local_token_mlp(tokens[:, 1:])                         # [(b v), (h w), c]
        c = global_token.shape[-1]
        global_token = global_token.reshape(b, v, c, 1, 1).expand(b, v, c, h, w)
        local_tokens = local_tokens.reshape(b, v, h // p, w // p, c).permute(0, 1, 4, 2, 3)
        local_tokens = local_tokens.repeat_interleave(p, dim=3).repeat_interleave(p, dim=4)
        return resnet_features + local_tokens + global_token

    @property
    def patch_size(self) -> int:
        return int("".join(filter(str.isdigit, self.cfg.model)))

    @property
    def d_out(self) -> int:
        return self.cfg.d_out


BACKBONES = {"resnet": BackboneResnet, "dino": BackboneDino}
BackboneCfg = BackboneResnetCfg | BackboneDinoCfg


def get_backbone(cfg: BackboneCfg, d_in: int) -> nn.Module:
    return BACKBONES[cfg.name](cfg, d_in)
