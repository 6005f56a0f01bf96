"""Videos on the GPU, on the tiny RE10k dataset of tests/dataset_golden.py with the re10k preset encoder and seeded
random weights:
  1. every video's Gaussians equal two full encoder calls per video in the reference's order, bit for bit;
  2. the colour panels equal the decoder's colour on the same 32-view chunks, quantised; the depth panels equal the
     turbo entries of `depth_color_index`, whose entries equal a float64 restatement of the reference's depth_map
     away from entry boundaries;
  3. two runs give the same frames;
  4. render-video writes readable MP4s for the 2-view and 3-view presets;
  5. a training run with --val-videos writes the videos and ends with the weights of the same run without them."""
import json
from dataclasses import replace

import numpy as np
import pytest
import torch

from pixelsplat_b200 import video
from pixelsplat_b200.data import device_shim
from pixelsplat_b200.encoder.encoder_tail import EncoderEpipolarTail
from pixelsplat_b200.evaluation import presets as ev
from pixelsplat_b200.evaluation.image_io import quantise
from pixelsplat_b200.evaluation.metrics import CHUNK
from tests import dataset_golden as dg
from tests import test_training_gpu as tt
from tests.test_training_gpu import deterministic  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
DEV = tt.DEV
INDEX = dg.DATA / "evaluation_index.json"
H = W = 256
X = {False: 8, True: 8 + W + 8}          # column of the probabilistic / deterministic panels
Y_COLOR, Y_DEPTH = 8, 8 + H + 8


def scene(preset: str = "re10k"):
    torch.manual_seed(0)
    cfg = ev.dataset_cfg(dg.DATA, INDEX, preset=preset)
    encoder, decoder = ev.build_model(preset, cfg)
    encoder, decoder = encoder.to(DEV).eval(), decoder.to(DEV)
    batch = next(iter(torch.utils.data.DataLoader(ev.make_test_dataset(cfg), batch_size=1, num_workers=0)))
    return encoder, decoder, encoder.get_data_shim()(device_shim(batch, (H, W), DEV))


def render_all(encoder, decoder, batch, seed=11, step=3):
    torch.manual_seed(seed)
    with torch.no_grad():
        features, _ = encoder.trunk(batch["context"])
        return {name: video.render_video(encoder, decoder, batch["context"], batch["target"], name, step, features,
                                         log=None) for name in video.VIDEOS}


EPS32 = torch.finfo(torch.float32).eps


def index64(depth: torch.Tensor):
    """The reference's depth_map restated in float64 on the same depth: the table entry, 256 x, and a bound on how far
    the float32 256 x can be from it (a few roundings of log d, of the quantiles and their logs, of the subtraction,
    the division and 1 - q, doubled); infinite where d = 0, whose x is clipped either way."""
    d = depth.double()
    near = d[d > 0][:video.QUANTILE_LIMIT].quantile(0.01).log()
    far = d.reshape(-1)[:video.QUANTILE_LIMIT].quantile(0.99).log()
    log = d.log()
    q = (log - near) / (far - near)
    x = (1 - q).clip(0, 1)
    e = 3 * EPS32
    span = (far - near).abs()
    dq = ((e * (log.abs() + 1) + e * (near.abs() + 1) + EPS32 * (log - near).abs()) / span
          + q.abs() * (e * (far.abs() + 1) + e * (near.abs() + 1) + EPS32 * span) / span + EPS32 * q.abs())
    bound = torch.where(log.isfinite(), 2 * 256 * (dq + EPS32), torch.inf)
    return torch.where(x.isnan(), 256, (x * 256).floor().clamp_max(255).long()), x * 256, bound


def test_frames_are_the_encoder_decoder_and_colour_rule(deterministic, monkeypatch):  # noqa: F811
    encoder, decoder, batch = scene()
    ctx, tgt = batch["context"], batch["target"]
    tails, forward = [], EncoderEpipolarTail.forward
    monkeypatch.setattr(EncoderEpipolarTail, "forward", lambda *a, **k: tails.append(forward(*a, **k)) or tails[-1])
    videos = render_all(encoder, decoder, batch)
    monkeypatch.setattr(EncoderEpipolarTail, "forward", forward)

    # the reference: two full encoder calls per video, probabilistic first, in the order rgb, wobble, exaggerated
    torch.manual_seed(11)
    with torch.no_grad():
        full = [encoder(ctx, 3, deterministic=d) for _ in video.VIDEOS for d in (False, True)]
    assert len(tails) == len(full) == 6
    for i, (a, b) in enumerate(zip(tails, full)):
        for field in ("means", "covariances", "harmonics", "opacities"):
            assert torch.equal(getattr(a, field), getattr(b, field)), (i, field)
    assert not torch.equal(full[0].means, full[2].means)           # each video draws its own depths

    table = torch.from_numpy(video.turbo_table()).to(DEV)
    for v, (name, frames) in enumerate(videos.items()):
        spec = video.VIDEOS[name]
        assert frames.dtype == torch.uint8 and frames.shape == (video.num_video_frames(name), 536, 536, 3), name
        if spec.loop_reverse:
            n = spec.num_frames
            assert torch.equal(frames[n:], torch.flip(frames[1:n - 1], [0])), name
        ext, k = (c.to(DEV)[None] for c in video.video_trajectory(ctx, tgt, name))
        t = ext.shape[1]
        near, far = ctx["near"][:, :1].expand(1, t).contiguous(), ctx["far"][:, :1].expand(1, t).contiguous()
        frames = frames[:t].to(DEV)
        for deterministic_tail in (False, True):
            g = full[2 * v + deterministic_tail]
            color, depth = [], []
            for i in range(0, t, CHUNK):
                out = decoder.forward(g, ext[:, i:i + CHUNK].contiguous(), k[:, i:i + CHUNK].contiguous(),
                                      near[:, i:i + CHUNK], far[:, i:i + CHUNK], (H, W), depth_mode="depth")
                color.append(out.color[0])
                depth.append(out.depth[0])
            color, depth = torch.cat(color), torch.cat(depth)
            x = X[deterministic_tail]
            assert torch.equal(frames[:, Y_COLOR:Y_COLOR + H, x:x + W], quantise(color)), (name, deterministic_tail)
            idx = video.depth_color_index(depth)
            assert torch.equal(frames[:, Y_DEPTH:Y_DEPTH + H, x:x + W], table[idx.clamp_max(255)]), name
            want, scaled, bound = index64(depth)
            inside = (scaled > 0) & (scaled < 256)            # clipped pixels get entry 0 or 255 either way
            gap = (scaled - scaled.round()).abs()
            within_1e5 = inside & (gap < 1e-5)
            flagged = inside & (gap < bound.clamp_min(1e-5))
            mismatched = int((idx != want)[~flagged].sum())
            print(f"{name} {'det' if deterministic_tail else 'prob'}: of {idx.numel()} pixels, {int(within_1e5.sum())} "
                  f"lie within 1e-5 of an entry boundary and {int(flagged.sum())} within the float32 bound "
                  f"(median {float(bound[inside].median()):.2e}); {int((idx != want)[flagged].sum())} of those and "
                  f"{mismatched} others differ; background {int((depth == 0).sum())}")
            assert mismatched == 0
            assert not (idx == 256).any()
        # the white gaps and border
        assert (frames[:, :8] == 255).all() and (frames[:, :, 8 + W:16 + W] == 255).all()


def test_two_runs_give_the_same_frames(deterministic):  # noqa: F811
    encoder, decoder, batch = scene()
    a, b = render_all(encoder, decoder, batch), render_all(encoder, decoder, batch)
    for name in video.VIDEOS:
        assert torch.equal(a[name], b[name]), name


def read_mp4(path):
    import cv2
    cap = cv2.VideoCapture(str(path))
    try:
        assert cap.isOpened(), path
        fps = cap.get(cv2.CAP_PROP_FPS)
        frames = []
        while True:
            ok, frame = cap.read()
            if not ok:
                break
            frames.append(frame)
    finally:
        cap.release()
    return np.stack(frames), fps


@pytest.mark.parametrize("preset", ["re10k", "re10k_3_view"])
def test_command_line_writes_readable_videos(preset, tmp_path):
    from pixelsplat_b200.evaluation import __main__ as cli
    from pixelsplat_b200.evaluation.checkpoint import save_checkpoint
    torch.manual_seed(0)
    encoder, _ = ev.build_model(preset, ev.dataset_cfg(dg.DATA, INDEX, preset=preset))
    ckpt = save_checkpoint(tmp_path / "random.ckpt", encoder, 0)
    scenes = [w["scene"] for w in dg.expected("test")]
    out = tmp_path / "videos"
    written = cli.render_videos(["--dataset-root", str(dg.DATA), "--index", str(INDEX), "--checkpoint", str(ckpt),
                                 "--preset", preset, "--num-workers", "0", "--output", str(out),
                                 "--scene", scenes[-1]])
    names = ["rgb.mp4", "wobble.mp4"] if preset == "re10k" else ["rgb.mp4"]
    assert sorted(p.name for p in written) == names
    assert sorted(p.name for p in (out / scenes[-1]).iterdir()) == names and len(list(out.iterdir())) == 1
    for p in written:
        frames, fps = read_mp4(p)
        assert frames.shape == (58 if p.stem == "rgb" else 118, 536, 536, 3) and fps == pytest.approx(30), p
    with pytest.raises(SystemExit, match="no test scene named zzz"):
        cli.main(["render-video", "--dataset-root", str(dg.DATA), "--index", str(INDEX), "--checkpoint", str(ckpt),
                  "--preset", preset, "--num-workers", "0", "--output", str(tmp_path / "none"), "--scene", "zzz"])


def test_training_with_val_videos_writes_them_and_keeps_the_weights(tmp_path, monkeypatch):
    from pixelsplat_b200.evaluation.checkpoint import read_checkpoint
    from pixelsplat_b200.lpips import Lpips
    from pixelsplat_b200.training import presets as tp
    from pixelsplat_b200.training.__main__ import main
    monkeypatch.setattr(Lpips, "from_files", classmethod(lambda cls, *a, **k: tt.seeded_lpips()))
    build_model = ev.build_model

    def conv_model(preset, cfg):
        # the one-convolution backbone: the DINO backbone's F.interpolate has no deterministic backward, so only
        # this model's training is bit-reproducible (test_training_gpu.py)
        encoder, decoder = build_model(preset, cfg)
        encoder.backbone = tt.ConvBackbone()
        return encoder, decoder

    monkeypatch.setattr(ev, "build_model", conv_model)
    monkeypatch.setitem(tp.TRAIN_PRESETS, "re10k", replace(tp.train_preset("re10k"), view_sampler=tt.TINY_SAMPLER))
    common = ["--dataset-root", str(dg.DATA), "--preset", "re10k", "--batch-size", "1", "--num-workers", "0",
              "--log-every", "1", "--val-every", "1", "--max-steps", "2", "--deterministic"]
    main(common + ["--output", str(tmp_path / "off")])
    main(common + ["--output", str(tmp_path / "on"), "--val-videos"])
    assert not (tmp_path / "off" / "validation" / "video").exists()
    for name, count in (("rgb", 58), ("wobble", 118)):
        files = sorted((tmp_path / "on" / "validation" / "video" / name).iterdir())
        assert [p.name for p in files] == [f"{s:0>6}.mp4" for s in (0, 1, 2)]
        for p in files:
            frames, _ = read_mp4(p)
            assert frames.shape == (count, 536, 536, 3)
    a = read_checkpoint(tmp_path / "off" / "checkpoints" / "epoch=0-step=2.ckpt")
    b = read_checkpoint(tmp_path / "on" / "checkpoints" / "epoch=0-step=2.ckpt")
    assert tt.state_equal(a["state_dict"], b["state_dict"])
    read = lambda p: [{k: v for k, v in json.loads(s).items() if k != "ms"} for s in p.read_text().splitlines()]
    assert read(tmp_path / "off" / "validation.jsonl") == read(tmp_path / "on" / "validation.jsonl")
