"""CPU tests of the image backbones and the whole encoder (pixelsplat_b200/encoder/backbone.py and
encoder_epipolar.py): state-dict keys and shapes against the reference modules' (tests/golden/backbone_keys.json,
written by oracle/make_backbone_golden.py), strict loading, weights from files without any download, DINO's
position-encoding resampling against a float64 restatement, and the argument checks of the ViT attention ABI."""
import ctypes
import json
import math
from pathlib import Path

import numpy as np
import pytest
import torch

GOLDEN = Path(__file__).resolve().parent / "golden"


def _keys(name):
    return {k: tuple(s) for k, s in json.loads((GOLDEN / "backbone_keys.json").read_text())[name]}


def _re10k_encoder_cfg():
    from pixelsplat_b200.encoder import EpipolarTransformerCfg, GaussianAdapterCfg, ImageSelfAttentionCfg
    from pixelsplat_b200.encoder.backbone import BackboneDinoCfg
    from pixelsplat_b200.encoder.encoder_epipolar import EncoderEpipolarCfg, OpacityMappingCfg
    return EncoderEpipolarCfg(
        name="epipolar", d_feature=128, num_monocular_samples=32, num_surfaces=1, predict_opacity=False,
        backbone=BackboneDinoCfg("dino", "dino_vitb8", 512), visualizer=None, near_disparity=3.0,
        gaussian_adapter=GaussianAdapterCfg(0.5, 15.0, 4), apply_bounds_shim=True,
        epipolar_transformer=EpipolarTransformerCfg(ImageSelfAttentionCfg(4, 10, 2, 4, 128, 128, 256),
                                                    10, 2, 4, 32, 128, 256, 4),
        opacity_mapping=OpacityMappingCfg(0.0, 0.0, 1), gaussians_per_pixel=3, use_epipolar_transformer=True,
        use_transmittance=False)


def _modules():
    from pixelsplat_b200.encoder.backbone import BackboneDino, BackboneDinoCfg, BackboneResnet, BackboneResnetCfg
    from pixelsplat_b200.encoder.encoder_epipolar import EncoderEpipolar
    return {
        "BackboneDino": lambda: BackboneDino(BackboneDinoCfg("dino", "dino_vitb8", 512), 3),
        "BackboneResnet": lambda: BackboneResnet(BackboneResnetCfg("resnet", "resnet50", 5, False, 512), 3),
        "EncoderEpipolar": lambda: EncoderEpipolar(_re10k_encoder_cfg(), num_context_views=2),
    }


@pytest.mark.parametrize("name", ["BackboneDino", "BackboneResnet", "EncoderEpipolar"])
def test_state_dict_keys_and_shapes_equal_the_reference(name):
    m = _modules()[name]()
    ours = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert ours == _keys(name)


@pytest.mark.parametrize("name", ["BackboneDino", "EncoderEpipolar"])
def test_reference_state_dict_loads_strictly(name):
    """A state dict with exactly the reference's keys and shapes loads with strict=True, and every value lands."""
    m = _modules()[name]()
    sd = {}
    for i, (k, shape) in enumerate(_keys(name).items()):
        ref = m.state_dict()[k]
        sd[k] = torch.full(shape, float(i % 97) / 97.0, dtype=ref.dtype) if ref.is_floating_point() \
            else torch.full(shape, i, dtype=ref.dtype)
    m.load_state_dict(sd, strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_child_modules_sit_at_the_top_level():
    m = _modules()["EncoderEpipolar"]()
    top = {k.split(".")[0] for k in m.state_dict()}
    assert top == {"backbone", "backbone_projection", "epipolar_transformer", "depth_predictor", "to_gaussians",
                   "high_resolution_skip"}
    assert m.sampler is m.epipolar_transformer.epipolar_sampler


def _no_network(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("network API called")
    monkeypatch.setattr(torch.hub, "load", refuse)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)
    monkeypatch.setattr(torch.hub, "download_url_to_file", refuse)


def test_from_files_by_name_and_by_path(tmp_path, monkeypatch):
    from pixelsplat_b200.encoder import backbone as bb
    _no_network(monkeypatch)
    hub = tmp_path / "hub"
    (hub / "checkpoints").mkdir(parents=True)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(hub))
    vit, res = bb.dino_vitb16(), bb.dino_resnet50()
    with torch.no_grad():
        for p in list(vit.parameters()) + list(res.parameters()):
            p.uniform_(-1, 1)
    res_sd = {k: v for k, v in res.state_dict().items() if not k.startswith("fc.")}
    torch.save(vit.state_dict(), hub / "checkpoints" / bb.DINO_FILES["dino_vitb16"])
    torch.save(res_sd, tmp_path / "my_resnet.pth")
    cfg = bb.BackboneDinoCfg("dino", "dino_vitb16", 64)
    # ViT by its released name in the hub directory, ResNet by explicit path
    m = bb.BackboneDino.from_files(cfg, 3, resnet_path=tmp_path / "my_resnet.pth")
    assert all(torch.equal(v, vit.state_dict()[k]) for k, v in m.dino.state_dict().items())
    assert all(torch.equal(v, res_sd[k]) for k, v in m.resnet_backbone.model.state_dict().items())
    # pretrained=True reads both from the hub directory
    torch.save(res_sd, hub / "checkpoints" / bb.DINO_FILES["dino_resnet50"])
    m2 = bb.BackboneDino(cfg, 3, pretrained=True)
    assert torch.equal(m2.dino.pos_embed, vit.pos_embed)
    assert torch.equal(m2.resnet_backbone.model.conv1.weight, res.conv1.weight)


def test_missing_weight_file_raises_and_names_it(tmp_path, monkeypatch):
    from pixelsplat_b200.encoder import backbone as bb
    _no_network(monkeypatch)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    cfg = bb.BackboneDinoCfg("dino", "dino_vitb8", 64)
    with pytest.raises(FileNotFoundError, match="dino_vitbase8_pretrain.pth"):
        bb.BackboneDino.from_files(cfg)
    with pytest.raises(FileNotFoundError, match="dino_resnet50"):
        bb.BackboneResnet(bb.BackboneResnetCfg("resnet", "dino_resnet50", 4, False, 64), 3, pretrained=True)
    with pytest.raises(FileNotFoundError, match="nowhere.pth"):
        bb.BackboneDino.from_files(cfg, vit_path=tmp_path / "nowhere.pth")


def test_modules_build_without_network(monkeypatch):
    from pixelsplat_b200.encoder import backbone as bb
    _no_network(monkeypatch)
    bb.get_backbone(bb.BackboneDinoCfg("dino", "dino_vitb16", 64), 3)
    bb.get_backbone(bb.BackboneResnetCfg("resnet", "resnet18", 4, False, 64), 3)


def _bicubic_f64(grid, out_h, out_w, scale_h, scale_w):
    """torch's bicubic (A = -0.75, align_corners=False, border clamp, source = (dst + 0.5) / scale - 0.5) in
    float64 numpy; grid [n, n, c]."""
    A = -0.75

    def weights(t):
        return np.array([((A * (t + 1) - 5 * A) * (t + 1) + 8 * A) * (t + 1) - 4 * A,
                         ((A + 2) * t - (A + 3)) * t * t + 1,
                         ((A + 2) * (1 - t) - (A + 3)) * (1 - t) * (1 - t) + 1,
                         ((A * (2 - t) - 5 * A) * (2 - t) + 8 * A) * (2 - t) - 4 * A])

    def matrix(n_out, n_in, scale):
        M = np.zeros((n_out, n_in))
        for i in range(n_out):
            src = (i + 0.5) / scale - 0.5
            x0 = math.floor(src)
            for j, w in enumerate(weights(src - x0)):
                M[i, min(max(x0 - 1 + j, 0), n_in - 1)] += w
        return M

    n = grid.shape[0]
    return np.einsum("ia,jb,abc->ijc", matrix(out_h, n, scale_h), matrix(out_w, n, scale_w), grid)


@pytest.mark.parametrize("hw", [(256, 256), (256, 192)])
def test_interpolate_pos_encoding_matches_float64(hw):
    from pixelsplat_b200.encoder import backbone as bb
    vit = bb.dino_vitb8()
    h, w = hw
    with torch.no_grad():
        tokens = vit.prepare_tokens(torch.zeros(1, 3, h, w))
    with torch.no_grad():
        got = vit.interpolate_pos_encoding(torch.zeros(1, 1 + (h // 8) * (w // 8), 768), h, w)
    pe = vit.pos_embed.detach().double().numpy()[0]
    n = int(math.sqrt(pe.shape[0] - 1))
    h0, w0 = h // 8 + 0.1, w // 8 + 0.1
    ref = _bicubic_f64(pe[1:].reshape(n, n, -1), h // 8, w // 8, h0 / n, w0 / n).reshape(-1, 768)
    assert got.shape == (1, 1 + (h // 8) * (w // 8), 768) and tokens.shape == got.shape
    assert np.array_equal(got[0, 0].double().numpy(), pe[0])
    # torch forms the source coordinates and cubic weights in fp32: measured 1.5e-6 at 256 x 192 on |values| < 0.1
    assert float(np.abs(got[0, 1:].double().numpy() - ref).max()) < 5e-6


# ---- the C ABI of the ViT attention kernel: rejections happen before any device work

P = ctypes.c_void_p(256)          # never dereferenced: every call below is rejected first
NUL = ctypes.c_void_p(0)


def _fwd(n=2, L=65, H=6, d=64, qkv=P, out=P, lse=P):
    from pixelsplat_b200 import _lib
    return _lib.lib.ps_vit_attention_forward(n, L, H, d, qkv, ctypes.c_float(0.125), out, lse, NUL)


def _bwd(n=2, L=65, H=6, d=64, ptrs=(P,) * 6, ws_bytes=None):
    from pixelsplat_b200 import _lib
    if ws_bytes is None:
        ws_bytes = n * H * max(L, 1) * 4
    qkv, out, dout, lse, dqkv, ws = ptrs
    return _lib.lib.ps_vit_attention_backward(n, L, H, d, qkv, out, dout, lse, ctypes.c_float(0.125), dqkv, ws,
                                              ws_bytes, NUL)


def test_vit_attention_rejects_bad_arguments():
    from pixelsplat_b200._lib import PS_ERR_UNSUPPORTED
    INVALID = 1
    assert _fwd(d=128) == PS_ERR_UNSUPPORTED and _bwd(d=32) == PS_ERR_UNSUPPORTED
    assert _fwd(L=0) == INVALID and _bwd(L=0) == INVALID
    assert _fwd(L=16385) == PS_ERR_UNSUPPORTED and _bwd(L=16385) == PS_ERR_UNSUPPORTED
    assert _fwd(H=17) == PS_ERR_UNSUPPORTED and _bwd(H=17) == PS_ERR_UNSUPPORTED
    assert _fwd(H=0) == INVALID and _fwd(n=0) == INVALID
    assert _fwd(qkv=NUL) == INVALID and _fwd(out=NUL) == INVALID and _fwd(lse=NUL) == INVALID
    for i in range(6):
        ptrs = [P] * 6
        ptrs[i] = NUL
        assert _bwd(ptrs=tuple(ptrs)) == INVALID
    assert _bwd(ws_bytes=2 * 6 * 65 * 4 - 1) == INVALID
    assert _fwd(qkv=ctypes.c_void_p(260)) == INVALID                 # not 16-byte aligned


def test_vit_attention_workspace_query():
    from pixelsplat_b200.encoder import vit_attention as va
    assert va.workspace_bytes(14, 1025, 12) == 14 * 12 * 1025 * 4
    with pytest.raises(Exception, match="PS_ERR_UNSUPPORTED"):
        va.workspace_bytes(1, 1025, 12, 128)


def test_attention_on_cpu_tensors_is_dinos_formula():
    """The kernel takes CUDA tensors only; a CPU module (checkpoint conversion, these tests) computes DINO's formula."""
    from pixelsplat_b200.encoder.backbone import Attention
    torch.manual_seed(0)
    a = Attention(128, 2)
    x = torch.randn(2, 9, 128)
    q, k, v = a.qkv(x).reshape(2, 9, 3, 2, 64).permute(2, 0, 3, 1, 4)
    ref = a.proj(((q @ k.transpose(-2, -1)) * 64 ** -0.5).softmax(-1).matmul(v).transpose(1, 2).reshape(2, 9, 128))
    assert torch.allclose(a(x), ref, atol=1e-6)
