"""GPU tests of the image backbones and the whole encoder against the reference modules' outputs
(tests/golden/backbone_v1.npz, written by oracle/make_backbone_golden.py with the same seeded weights; it stores a
subsample of each float64 result and the reference's own fp32-vs-float64 error on that subsample).

Bar, in the style of test_adapter_gpu.py: relative max-norm error against the reference's float64 run at most
4x the reference's own fp32-vs-float64 error plus a ceiling; cuDNN's TF32 convolutions are turned off.
  - Outputs, and everything with DINO's explicit fp32 attention (PIXELSPLAT_B200_VIT_ATTENTION=fp32): the ceiling
    is 2e-3 with the TF32 attention kernel (csrc/vit_attention.cu, 2e-3 on its own) and 2e-5 without it.  This
    pins the wiring tightly: measured <= 1.5e-5 on the fp32 route.
  - Gradients that flow back through the ViT's attention with the kernel: 5e-2.  With seeded random weights the
    attention is close to uniform, so dP - D in dS = P (dP - D) is a small difference of TF32 products and dQ, dK
    keep only a few digits; over 12 blocks that reaches 3.1e-2 on the image gradient and 1.3e-2 on the patch
    embedding (measured on an H100), while the same run meets 2e-5 on the fp32 route.
The InstanceNorm ResNet's image gradient is ill-conditioned at 64 x 64 (layer4 normalises 2 x 2 maps): the
reference's own fp32 run is 4.2e-2 from float64 there, and the bar scales with it.
"""
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = np.load(Path(__file__).resolve().parent / "golden" / "backbone_v1.npz")
CEIL_TF32, CEIL_FP32, CEIL_TF32_GRAD = 2e-3, 2e-5, 5e-2


@pytest.fixture(autouse=True)
def _no_tf32_convolutions():
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


def _check(got, name, ceil):
    from oracle.make_backbone_golden import rel_err
    ref = GOLD[name].astype(np.float64)
    assert got.shape == ref.shape
    err, bar = rel_err(got, ref), 4 * float(GOLD[name + "_f32_err"]) + ceil
    assert err <= bar, f"{name}: {err:.2e} > {bar:.2e}"


def _run(module, name, ceil_out, ceil_grad):
    from oracle.make_backbone_golden import images, loss_weights, sub, sub_image
    module = module.to(DEV).eval()
    x = images((1, 2, 3, 64, 64), 1).float().to(DEV).requires_grad_(True)
    y = module({"image": x})
    (y * loss_weights(y.shape, name).float().to(DEV)).sum().backward()
    _check(sub(y.detach()).double().cpu().numpy(), name + "_out", ceil_out)
    _check(sub_image(x.grad).double().cpu().numpy(), name + "_d_image", ceil_grad)
    return module


def test_backbone_resnet_matches_the_reference():
    from oracle.make_backbone_golden import seeded_state_dict
    from pixelsplat_b200.encoder.backbone import BackboneResnet, BackboneResnetCfg
    m = BackboneResnet(BackboneResnetCfg("resnet", "resnet50", 5, False, 512), 3)
    m.load_state_dict(seeded_state_dict(m, 0))
    _run(m, "resnet", CEIL_FP32, CEIL_FP32)


@pytest.mark.parametrize("route", ["tf32", "fp32"])
def test_backbone_dino_matches_the_reference(route, monkeypatch):
    from oracle.make_backbone_golden import PARAM_SLICE, PARAM_SLICES, seeded_state_dict
    from pixelsplat_b200.encoder.backbone import BackboneDino, BackboneDinoCfg
    monkeypatch.setenv("PIXELSPLAT_B200_VIT_ATTENTION", route)
    ceil_out, ceil_grad = (CEIL_TF32, CEIL_TF32_GRAD) if route == "tf32" else (CEIL_FP32, CEIL_FP32)
    m = BackboneDino(BackboneDinoCfg("dino", "dino_vitb8", 512), 3)
    m.load_state_dict(seeded_state_dict(m, 1))
    m = _run(m, "dino", ceil_out, ceil_grad)
    params = dict(m.named_parameters())
    for k in PARAM_SLICES:
        through_vit = k.startswith("dino.")
        _check(params[k].grad.double().reshape(-1)[:PARAM_SLICE].cpu().numpy(), "dino_d_" + k,
               ceil_grad if through_vit else ceil_out)


def test_vit_at_1025_tokens_matches_the_reference():
    from oracle.make_backbone_golden import images, seeded_state_dict, sub_tokens
    from pixelsplat_b200.encoder.backbone import dino_vitb8
    vit = dino_vitb8()
    vit.load_state_dict(seeded_state_dict(vit, 2))
    vit = vit.to(DEV)
    with torch.no_grad():
        tok = vit.get_intermediate_layers(images((1, 3, 256, 256), 2).float().to(DEV))[0]
    assert tok.shape == (1, 1025, 768)
    _check(sub_tokens(tok).double().cpu().numpy(), "vit256_tokens", CEIL_TF32)


def test_encoder_to_decoder_end_to_end():
    """EncoderEpipolar (dino_vitb8 backbone, the re10k encoder) -> DecoderSplattingCUDA.forward_mse, forward and
    backward: finite loss and a finite gradient on every parameter the reference's forward uses (BackboneDino runs
    DINO's ResNet-50 through layer3 only, so its layer4 gets no gradient there either)."""
    from pixelsplat_b200.decoder import DecoderSplattingCUDA, DecoderSplattingCUDACfg
    from pixelsplat_b200.encoder.encoder_epipolar import EncoderEpipolar
    from tests import golden_util as gu
    from tests.test_backbone_cpu import _re10k_encoder_cfg
    torch.manual_seed(0)
    enc = EncoderEpipolar(_re10k_encoder_cfg(), num_context_views=2).to(DEV)
    ext, K, near, far = [t.to(DEV, torch.float32) for t in gu.camera_rig(1, 2, "generic")]
    image = torch.rand(1, 2, 3, 64, 64, device=DEV)
    gs = enc(dict(image=image, extrinsics=ext, intrinsics=K, near=near, far=far), global_step=0)
    dec = DecoderSplattingCUDA(DecoderSplattingCUDACfg("splatting_cuda"),
                               type("D", (), {"background_color": [0.0, 0.0, 0.0]})()).to(DEV)
    _, sse, _ = dec.forward_mse(gs, ext, K, near, far, (64, 64), image)
    sse.sum().backward()
    torch.cuda.synchronize()
    assert torch.isfinite(sse).all() and gs.means.shape == (1, 2 * 64 * 64 * 3, 3)
    for name, p in enc.named_parameters():
        if name.startswith("backbone.resnet_backbone.model.layer4."):
            assert p.grad is None
            continue
        assert p.grad is not None and torch.isfinite(p.grad).all(), name
