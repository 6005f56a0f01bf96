"""GPU tests of the evaluation: the frame pass of csrc/eval_images.cu against torch's prep_image route and the PNG
round trip, frame_metrics against the reference's metric route restated in float64, and the evaluator and metric
computer end to end on the tiny RE10k dataset of tests/dataset_golden.py."""
import json

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import lpips_oracle as lo
from oracle import ssim_oracle
from pixelsplat_b200 import _lib
from pixelsplat_b200.decoder import DecoderSplattingCUDA, DecoderSplattingCUDACfg, Gaussians
from pixelsplat_b200.evaluation import (Evaluator, Method, compute_metrics, frame_metrics, frame_pass, load_checkpoint,
                                        load_image, prep_image, save_image)
from pixelsplat_b200.evaluation.presets import build_model
from pixelsplat_b200.loss import compute_psnr
from pixelsplat_b200.lpips import Lpips
from pixelsplat_b200 import synthetic
from tests import dataset_golden as dg
from tests.test_evaluation_cpu import crafted_image, crafted_values

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def torch_route(x: torch.Tensor):
    """prep_image's quantisation on the device and ToTensor's dequantisation on the host, where the reference's
    load_image runs it: (uint8 [n, h, w, 3], float32 planes).  (torch on CUDA divides by a host scalar as a
    multiplication by its reciprocal, which is not u / 255 for every u; ToTensor on the host divides.)"""
    u = (x.clip(min=0, max=1) * 255).to(torch.uint8)
    return u.permute(0, 2, 3, 1).contiguous(), (u.cpu().float() / 255).to(x.device)


def sse_f64(planes: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    return ((planes.double() - target.clip(0, 1).double()) ** 2).sum(dim=(1, 2, 3))


def _decoder():
    return DecoderSplattingCUDA(DecoderSplattingCUDACfg("splatting_cuda"),
                                type("D", (), {"background_color": [0.0, 0.0, 0.0]})()).to(DEV)


def rendered(kind: str) -> torch.Tensor:
    """Renders of configs[0] (64 x 64, one view) or of a re10k-like 256 x 256 scene (four target views)."""
    sc = synthetic.scene_random_frustum(seed=0) if kind == "configs0" else \
        synthetic.scene_re10k_like(seed=0, target_views=4)
    g = Gaussians(*(t.to(DEV)[None] for t in (sc.means, sc.covariances, sc.harmonics, sc.opacities)))
    with torch.no_grad():
        return _decoder()(g, sc.extrinsics.to(DEV)[None], sc.intrinsics.to(DEV)[None], sc.near.to(DEV)[None],
                          sc.far.to(DEV)[None], sc.image_shape).color[0]


def inputs(kind: str, n: int):
    """(renders, targets) float32 [n, 3, h, w]."""
    g = torch.Generator().manual_seed(n)
    if kind == "crafted":
        x = torch.stack([crafted_image(19, 37, seed=i) for i in range(n)])
    elif kind == "random":
        x = torch.rand(n, 3, 40, 56, generator=g) * 1.4 - 0.2
    else:
        r = rendered(kind)
        x = r[torch.arange(n) % r.shape[0]].cpu()
    t = (x + 0.1 * torch.randn(x.shape, generator=g)).nan_to_num(0.5)
    return x.to(DEV), t.to(DEV)


@pytest.mark.parametrize("kind", ["crafted", "random", "configs0", "re10k_like"])
@pytest.mark.parametrize("n", [1, 7, 32, 45])
def test_render_mode_equals_the_torch_route(kind, n):
    x, t = inputs(kind, n)
    fp = frame_pass(x, target=t)
    want_u, want_planes = torch_route(x)
    assert torch.equal(fp.frames, want_u) and torch.equal(fp.planes, want_planes)
    err = ((fp.sse - sse_f64(want_planes, t)).abs() / sse_f64(want_planes, t)).max().item()
    assert err < 1e-6, err


def test_nan_maps_to_zero_and_inf_saturates():
    x = torch.tensor([float("nan"), float("inf"), -float("inf"), -0.0, 2.0, 0.5], device=DEV)
    fp = frame_pass(x.reshape(1, 3, 1, 2), target=torch.zeros(1, 3, 1, 2, device=DEV))
    # CHW planes (nan, inf), (-inf, -0), (2, 0.5) -> HWC pixels (0, 0, 255), (255, 0, 127)
    assert fp.frames.reshape(-1).tolist() == [0, 0, 255, 255, 0, 127]
    assert fp.sse.item() == pytest.approx(2.0 + (127 / 255) ** 2, rel=1e-7)


def test_frame_mode_equals_totensor_of_the_png(tmp_path):
    x, t = inputs("crafted", 5)
    for i in range(5):
        save_image(x[i], tmp_path / f"{i}.png")
    frames = torch.from_numpy(np.stack([np.array(Image.open(tmp_path / f"{i}.png")) for i in range(5)])).to(DEV)
    fp = frame_pass(frames, target=t)
    want = torch.stack([torch.from_numpy(np.array(Image.open(tmp_path / f"{i}.png"))).permute(2, 0, 1).float()
                        .div(255) for i in range(5)]).to(DEV)
    assert fp.frames is None and torch.equal(fp.planes, want)
    assert torch.equal(fp.sse, frame_pass(x, target=t).sse)          # the same sums from the frames as the renders
    assert torch.equal(load_image(tmp_path / "3.png"), want[3])
    assert np.array_equal(prep_image(x[2]), np.array(Image.open(tmp_path / "2.png")))


def test_prep_image_shapes_match_the_reference():
    x = torch.rand(2, 3, 8, 9, device=DEV) * 1.2 - 0.1
    ref = lambda im: (im.clip(0, 1) * 255).type(torch.uint8).permute(1, 2, 0).cpu().numpy()
    assert np.array_equal(prep_image(x), ref(x.permute(1, 2, 0, 3).reshape(3, 8, 18)))
    assert np.array_equal(prep_image(x[0, 0]), ref(x[0, :1].expand(3, -1, -1)))
    rgba = torch.cat([x[0], x[1, :1]])
    assert np.array_equal(prep_image(rgba), ref(rgba))


def test_psnr_within_a_ten_thousandth_of_a_db_and_inf_for_identical():
    x, t = inputs("re10k_like", 8)
    fp = frame_pass(x, target=t)
    h, w = x.shape[-2:]
    from pixelsplat_b200.evaluation import psnr_from_sse
    ours = psnr_from_sse(fp.sse, h, w)
    ref = compute_psnr(t, torch_route(x)[1])                          # the reference's float32 route
    assert (ours - ref).abs().max().item() < 1e-4
    same = torch_route(x)[1]
    assert torch.isinf(psnr_from_sse(frame_pass(x, target=same).sse, h, w)).all()


def test_repeated_runs_and_graph_replay_give_the_same_bits():
    x, t = inputs("random", 32)
    first = frame_pass(x, target=t)
    for _ in range(3):
        again = frame_pass(x, target=t)
        assert torch.equal(again.sse, first.sse) and torch.equal(again.planes, first.planes)
    frame_pass(x, target=t)                                            # warm-up outside the capture
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = frame_pass(x, target=t)
    for _ in range(2):
        captured.sse.zero_()
        captured.planes.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(captured.sse, first.sse) and torch.equal(captured.planes, first.planes)
        assert torch.equal(captured.frames, first.frames)


def test_frame_metrics_equal_the_reference_route(tmp_path):
    """PSNR / SSIM / LPIPS of the 8-bit frames against the round trip scored by the reference's formulas in
    float64 (seeded LPIPS weights).  Measured on the H100: see DESIGN section 6."""
    r = rendered("re10k_like")[:, :, 64:160, 64:160].contiguous()
    g = torch.Generator().manual_seed(3)
    gt = (r + 0.05 * torch.randn(r.shape, generator=g).to(DEV)).clamp(0, 1)
    sd = lo.random_state_dict(0)
    lp = Lpips()
    lp.load_state_dict(sd)
    lp = lp.to(DEV)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        got = frame_metrics(gt, r, lpips=lp)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    planes = []
    for i in range(r.shape[0]):
        save_image(r[i], tmp_path / f"{i}.png")
        planes.append(torch.from_numpy(np.array(Image.open(tmp_path / f"{i}.png"))).permute(2, 0, 1).float() / 255)
    planes = torch.stack(planes).double()
    gt64 = gt.double().cpu()
    psnr = -10 * ((gt64.clip(0, 1) - planes) ** 2).mean(dim=(1, 2, 3)).log10()
    ssim = ssim_oracle.ssim_numpy(gt64.numpy(), planes.numpy())
    lpips = lo.lpips(gt64, planes, {k: v.double() for k, v in sd.items()}, normalize=True)[:, 0, 0, 0]
    e_psnr = (got["psnr"].double().cpu() - psnr).abs().max().item()
    e_ssim = float(np.abs(got["ssim"].double().cpu().numpy() - ssim).max())
    e_lpips = ((got["lpips"].double().cpu() - lpips).abs() / lpips.abs()).max().item()
    print(f"frame_metrics vs float64 route: psnr {e_psnr:.2e} dB, ssim {e_ssim:.2e}, lpips {e_lpips:.2e} rel")
    assert e_psnr <= 1e-4 and e_ssim <= 1e-5 and e_lpips <= 1e-5


class _FixedEncoder(torch.nn.Module):
    """An encoder stand-in that returns fixed Gaussians and has an identity data shim."""

    def __init__(self, gaussians):
        super().__init__()
        self.gaussians = gaussians

    def get_data_shim(self):
        return lambda batch: batch

    def forward(self, context, global_step, deterministic=False):
        return self.gaussians


def test_seventy_targets_render_in_chunks_of_32():
    sc = synthetic.scene_random_frustum(seed=1)
    g = Gaussians(*(t.to(DEV)[None] for t in (sc.means, sc.covariances, sc.harmonics, sc.opacities)))
    ext = synthetic.target_cameras(70, seed=2).to(DEV)[None]
    K = sc.intrinsics[:1].to(DEV).expand(1, 70, 3, 3)
    near, far = sc.near[:1].to(DEV).expand(1, 70), sc.far[:1].to(DEV).expand(1, 70)
    dec = _decoder()
    calls = []
    forward = dec.forward

    def spy(gs, e, *a, **k):
        calls.append(e.shape[1])
        return forward(gs, e, *a, **k)

    dec.forward = spy
    target = torch.rand(1, 70, 3, 64, 64, device=DEV)
    batch = {"scene": ["s"], "context": {"index": torch.tensor([[0, 1]])},
             "target": {"extrinsics": ext, "intrinsics": K, "near": near, "far": far, "image": target,
                        "index": torch.arange(70)[None]}}
    r = Evaluator(_FixedEncoder(g), dec, lpips=_seeded_lpips()).test_step(batch)
    assert calls == [32, 32, 6]
    dec.forward = forward
    with torch.no_grad():
        color = torch.cat([dec(g, ext[:, i:j], K[:, i:j], near[:, i:j], far[:, i:j], (64, 64)).color[0]
                           for i, j in ((0, 32), (32, 64), (64, 70))])
    assert torch.equal(r.frames, torch_route(color)[0])
    assert r.per_view["psnr"].shape == (70,)


def _seeded_lpips():
    lp = Lpips()
    lp.load_state_dict(lo.random_state_dict(0))
    return lp.to(DEV)


def _test_loader():
    return torch.utils.data.DataLoader(dg.dataset("test"), batch_size=1, num_workers=0)


def _lightning_checkpoint(path, encoder):
    torch.save({"epoch": 0, "global_step": 17, "state_dict": {f"encoder.{k}": v for k, v in
                                                               encoder.state_dict().items()}}, path)


def test_evaluator_and_metric_computer_end_to_end(tmp_path, monkeypatch):
    cfg = dg.dataset("test").cfg
    torch.manual_seed(0)
    seeded, _ = build_model("re10k", cfg)
    _lightning_checkpoint(tmp_path / "m.ckpt", seeded)
    encoder, decoder = build_model("re10k", cfg)
    assert load_checkpoint(tmp_path / "m.ckpt", encoder) == 17
    encoder, decoder = encoder.to(DEV).eval(), decoder.to(DEV)
    lp = _seeded_lpips()
    out = tmp_path / "ours"
    res = Evaluator(encoder, decoder, out, lpips=lp).run(_test_loader(), (256, 256), keep_frames=True, log=None)

    # the scenes, contexts and targets of the reference's test split (fff has no index entry and is skipped)
    want = dg.expected("test")
    assert [(s.scene, s.context_index, s.target_index) for s in res.scenes] == \
        [(w["scene"], w["context"]["index"].tolist(), w["target"]["index"].tolist()) for w in want]
    for s in res.scenes:
        for i, index in enumerate(s.target_index):
            png = np.array(Image.open(out / s.scene / "color" / f"{index:0>6}.png"))
            assert np.array_equal(png, s.frames[i].cpu().numpy())
        for index in s.context_index:
            assert (out / s.scene / "context" / f"{index:0>6}.png").is_file()
        assert all(np.isfinite(v) for v in s.metrics.values())
    bench = json.loads((out / "benchmark.json").read_text())
    assert len(bench["encoder"]) == 2 and len(bench["decoder"]) == sum(len(s.target_index) for s in res.scenes)
    assert json.loads((out / "peak_memory.json").read_text()) > 0

    # a "method" whose frames are the ground truth
    gt_dir = tmp_path / "gt"
    from pixelsplat_b200.data import device_shim
    for b in _test_loader():
        b = device_shim(b, (256, 256))
        for index, img in zip(b["target"]["index"][0].tolist(), b["target"]["image"][0]):
            save_image(img, gt_dir / b["scene"][0] / "color" / f"{index:0>6}.png")

    methods = [Method("Ours", "ours", out), Method("Truth", "gt", gt_dir)]
    mc = compute_metrics(methods, _test_loader(), lpips=lp, log=None)
    assert mc.skipped == [] and list(mc.scenes) == [s.scene for s in res.scenes]
    for s in res.scenes:
        for k in ("psnr", "ssim", "lpips"):
            assert mc.scenes[s.scene][f"{k}_ours"] == s.metrics[k], (s.scene, k)
        assert mc.scenes[s.scene]["psnr_gt"] == float("inf") and mc.scenes[s.scene]["lpips_gt"] == 0.0
        assert abs(mc.scenes[s.scene]["ssim_gt"] - 1.0) < 1e-6
    for k in ("psnr", "ssim", "lpips"):
        assert mc.mean[f"{k}_ours"] == res.mean[k]

    # a missing frame skips the scene
    (gt_dir / res.scenes[0].scene / "color" / f"{res.scenes[0].target_index[0]:0>6}.png").unlink()
    mc2 = compute_metrics(methods, _test_loader(), lpips=lp, log=None)
    assert mc2.skipped == [res.scenes[0].scene] and list(mc2.scenes) == [s.scene for s in res.scenes[1:]]

    # deterministic encoder under torch's deterministic algorithms: two runs, the same metrics
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    try:
        runs = [Evaluator(encoder, decoder, lpips=lp, deterministic=True).run(_test_loader(), (256, 256), log=None)
                for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(False)
    assert [s.metrics for s in runs[0].scenes] == [s.metrics for s in runs[1].scenes]
    assert runs[0].mean == runs[1].mean


def test_shim_that_changes_the_targets_raises():
    cfg = dg.dataset("test").cfg
    encoder, decoder = build_model("re10k", cfg)
    ev = Evaluator(encoder.to(DEV), decoder.to(DEV), lpips=_seeded_lpips())
    from pixelsplat_b200.data import device_shim
    batch = device_shim(next(iter(_test_loader())), (180, 320))       # 180 is not a multiple of 16
    with pytest.raises(ValueError, match="data shim changed the targets"):
        ev.test_step(batch)


def test_crafted_values_cover_the_truncation_edges():
    v = torch.from_numpy(crafted_values()).to(DEV)
    n = v.numel() // 3 * 3
    x = v[:n].reshape(1, 3, 1, -1)
    assert torch.equal(frame_pass(x).frames, torch_route(x)[0])
