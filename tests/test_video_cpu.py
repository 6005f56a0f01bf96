"""Videos without a GPU: the trajectories against the reference's own functions (tests/golden/video_trajectories_v1.npz,
oracle/make_video_golden.py), the time bases and frame counts, the frame layout, the depth colour index rule, an MP4
round trip and the command lines."""
import math

import numpy as np
import pytest
import torch

from pixelsplat_b200 import video
from pixelsplat_b200.evaluation.image_io import comparison_layout
from tests import dataset_golden as dg

GOLDEN = np.load(dg.GOLDEN / "video_trajectories_v1.npz")
CASES = [c for c in dict.fromkeys(k.split("/")[0] for k in GOLDEN.files if "/" in k) if c not in ("batch", "circular")]
# worst measured |ours - reference| / the pair's camera-position scale over every case: 0 (the same op order gives
# the same bits on the CPU); the bar is the one the trajectories are held to
BAR = 1e-6


def g(key: str) -> torch.Tensor:
    return torch.from_numpy(GOLDEN[key])


def scale(case: str) -> float:
    return max(1.0, float(g(f"{case}/initial")[:3, 3].norm()), float(g(f"{case}/final")[:3, 3].norm()))


def assert_close(got: torch.Tensor, want: torch.Tensor, s: float, what) -> float:
    assert got.dtype == want.dtype and got.shape == want.shape, what
    err = float((got.double() - want.double()).abs().max()) / s
    assert err <= BAR, (what, err)
    return err


def test_golden_covers_the_cases():
    assert set(CASES) == {"general", "parallel", "anti_parallel", "replaced_b", "yaw_wrap_left", "yaw_wrap_right",
                          "near_gimbal_pitch", "anisotropic"}


@pytest.mark.parametrize("case", CASES)
def test_trajectories_equal_the_reference(case):
    e0, e1, k0, k1 = (g(f"{case}/{k}") for k in ("initial", "final", "k0", "k1"))
    t_rgb, t_wobble, t_ex, t_5 = (g(k) for k in ("t_rgb", "t_wobble", "t_exaggerated", "t_exaggerated_5t_minus_2"))
    s = scale(case)
    delta = (e0[:3, 3] - e1[:3, 3]).norm(dim=-1)
    tf = video.generate_wobble_transformation(delta * 0.5, t_ex, 5, scale_radius_with_t=False)
    errs = [
        assert_close(video.interpolate_extrinsics(e0, e1, t_rgb), g(f"{case}/rgb_extrinsics"), s, "rgb"),
        assert_close(video.interpolate_intrinsics(k0, k1, t_rgb), g(f"{case}/rgb_intrinsics"), 1.0, "rgb K"),
        assert_close(tf, g(f"{case}/exaggerated_tf"), s, "exaggerated tf"),
        assert_close(video.interpolate_extrinsics(e0, e1, t_5) @ tf, g(f"{case}/exaggerated_extrinsics"), s,
                     "exaggerated"),
        assert_close(video.interpolate_intrinsics(k0, k1, t_5), g(f"{case}/exaggerated_intrinsics"), 1.0,
                     "exaggerated K"),
        assert_close(video.generate_wobble_transformation(delta * 0.25, t_wobble), g(f"{case}/wobble_tf"), s,
                     "wobble tf"),
        assert_close(video.generate_wobble(e0, delta * 0.25, t_wobble), g(f"{case}/wobble_extrinsics"), s, "wobble"),
    ]
    print(f"{case}: worst relative difference {max(errs):.3g}")


def test_batched_calls_broadcast_as_the_reference():
    e0 = torch.stack([g(f"{c}/initial") for c in CASES])
    e1 = torch.stack([g(f"{c}/final") for c in CASES])
    got = video.interpolate_extrinsics(e0, e1, g("t_rgb"))
    assert got.shape == (len(CASES), 30, 4, 4)
    s = max(scale(c) for c in CASES)
    assert_close(got, g("batch/extrinsics"), s, "batch")
    radius = (e0[:, :3, 3] - e1[:, :3, 3]).norm(dim=-1)
    assert_close(video.generate_wobble(e0, radius * 0.25, g("t_wobble")), g("batch/wobble"), s, "wobble")


def test_interpolate_circular_takes_every_branch_as_the_reference():
    a, b, t = g("circular/a"), g("circular/b"), g("circular/t")
    got = video._interpolate_circular(a, b, t)
    assert torch.equal(got, g("circular/result"))
    tau = 2 * math.pi
    am, bm = a % tau, b % tau
    d, dl, dr = (bm - am).abs(), (bm - am + tau).abs(), (bm - am - tau).abs()
    direct = (d < dl) & (d < dr)
    left = (dl < dr) & ~direct
    assert direct.any() and left.any() and (~direct & ~left).any()


def test_time_bases_and_frame_counts():
    for name, key in (("rgb", "t_rgb"), ("wobble", "t_wobble"), ("interpolation_exagerrated", "t_exaggerated")):
        spec = video.VIDEOS[name]
        assert torch.equal(video.time_steps(spec.num_frames, spec.smooth), g(key)), name
    assert torch.equal(video.time_steps(300, False) * 5 - 2, g("t_exaggerated_5t_minus_2"))
    assert [video.num_video_frames(n) for n in ("rgb", "wobble", "interpolation_exagerrated")] == [58, 118, 300]
    t = video.time_steps(30, True)
    assert t[0] == 0 and t[-1] == 1 and (t[1:] >= t[:-1]).all()


def batch_of(case: str, views: int = 2):
    e = torch.stack([g(f"{case}/initial"), g(f"{case}/final"), g(f"{case}/initial")])[:views]
    k = torch.stack([g(f"{case}/k0"), g(f"{case}/k1"), g(f"{case}/k0")])[:views]
    context = {"extrinsics": e[None], "intrinsics": k[None]}
    target = {"extrinsics": g(f"{case}/final")[None, None], "intrinsics": g(f"{case}/k1")[None, None]}
    return context, target


def test_video_cameras_are_the_reference_trajectories():
    context, target = batch_of("anisotropic")
    ext, k = video.video_trajectory(context, target, "rgb")
    assert torch.equal(ext, video.interpolate_extrinsics(context["extrinsics"][0, 0], context["extrinsics"][0, 1],
                                                         g("t_rgb")))
    assert torch.equal(k, g("anisotropic/rgb_intrinsics"))
    ext, k = video.video_trajectory(context, target, "wobble")
    assert torch.equal(ext, g("anisotropic/wobble_extrinsics")) and ext.shape == (60, 4, 4)
    assert torch.equal(k, context["intrinsics"][0, 0].expand(60, 3, 3))
    ext, k = video.video_trajectory(context, target, "interpolation_exagerrated")
    assert torch.equal(ext, g("anisotropic/exaggerated_extrinsics")) and k.shape == (300, 3, 3)
    # three context views: rgb ends at target 0, the other two are skipped
    context3, _ = batch_of("anisotropic", 3)
    target3 = {"extrinsics": g("general/final")[None, None], "intrinsics": g("general/k1")[None, None]}
    ext, _ = video.video_trajectory(context3, target3, "rgb")
    assert torch.equal(ext, video.interpolate_extrinsics(context3["extrinsics"][0, 0], g("general/final"),
                                                         g("t_rgb")))
    assert video.video_trajectory(context3, target3, "wobble") is None
    assert video.video_trajectory(context3, target3, "interpolation_exagerrated") is None


def test_layout_of_a_video_frame():
    t, h, w = 3, 16, 12
    panels = [torch.full((t, 3, h, w), v, dtype=torch.uint8) for v in (10, 20, 30, 40)]
    out = comparison_layout((panels[0], panels[1]), (panels[2], panels[3]))
    assert out.shape == (t, 3, 8 + 2 * h + 8 + 8, 8 + 2 * w + 8 + 8) and out.dtype == torch.uint8
    assert (out[..., 8:8 + h, 8:8 + w] == 10).all() and (out[..., 16 + h:16 + 2 * h, 8:8 + w] == 20).all()
    assert (out[..., 8:8 + h, 16 + w:16 + 2 * w] == 30).all()
    assert (out[..., 16 + h:16 + 2 * h, 16 + w:16 + 2 * w] == 40).all()
    inside = torch.zeros(out.shape[-2:], dtype=torch.bool)
    for y in (8, 16 + h):
        for x in (8, 16 + w):
            inside[y:y + h, x:x + w] = True
    assert (out[..., ~inside] == 255).all()
    # 256 x 256 panels give the reference's 536 x 536 frame
    p = torch.zeros(1, 3, 256, 256, dtype=torch.uint8)
    assert comparison_layout((p, p), (p, p)).shape == (1, 3, 536, 536)


def reference_index(depth: torch.Tensor) -> torch.Tensor:
    """The colour rule restated in float64 from the same float32 near / far."""
    near = depth[depth > 0][:video.QUANTILE_LIMIT].quantile(0.01).log()
    far = depth.reshape(-1)[:video.QUANTILE_LIMIT].quantile(0.99).log()
    x = (1 - (depth.double().log() - near.double()) / (far.double() - near.double())).clip(0, 1)
    return torch.where(x.isnan(), 256, (x * 256).floor().clamp_max(255).long())


def test_colour_index_rule():
    g_ = torch.Generator().manual_seed(0)
    d = torch.rand(4, 32, 32, generator=g_) * 10 + 0.1
    d[0, 0, :5] = 0                                       # background
    idx = video.depth_color_index(d)
    assert idx.dtype == torch.long and idx.shape == d.shape
    assert (idx[0, 0, :5] == 255).all()                   # log 0 = -inf -> x = 1 -> the last entry
    assert torch.equal(idx, reference_index(d))
    assert int(idx.min()) == 0 and int(idx.max()) == 255
    # a constant depth: far = near, so (log d - near) / 0 is NaN (black) on it and -inf -> entry 255 on background
    d = torch.full((2, 4, 4), 3.0)
    d[0, 0] = 0
    idx = video.depth_color_index(d)
    assert (idx[0, 0] == 255).all() and (idx[0, 1:] == 256).all() and (idx[1] == 256).all()
    # a NaN depth makes both quantiles NaN, as in the reference: every pixel is black
    d = torch.rand(2, 4, 4, generator=g_) + 1
    d[1, 2, 3] = float("nan")
    assert (video.depth_color_index(d) == 256).all()


def test_colour_index_on_exact_boundaries():
    # near = log 1, far = log e^2: x = 1 - log(d) / 2, so d = exp(2 (1 - k / 256)) puts x near k / 256; the entry is
    # floor(256 x) of the float32 x, whatever side of k / 256 it lands on
    k = torch.arange(0, 257, dtype=torch.float32)
    d = torch.cat([torch.ones(200), torch.exp(2 * (1 - k / 256)), torch.full((200,), math.exp(2))])
    idx = video.depth_color_index(d)
    near = d[d > 0].quantile(0.01).log()
    far = d.quantile(0.99).log()
    x = (1 - (d.log() - near) / (far - near)).clip(0, 1)
    assert torch.equal(idx, (x * 256).long().clamp_max(255))
    assert idx[200 + 256] == 255                          # x = 0 ... 1 both ends
    # exactly representable x = k / 256 lands on entry k (256 -> 255)
    x = torch.tensor([0.0, 1 / 256, 0.5, 255 / 256, 1.0])
    assert ((x * 256).long().clamp_max(255)).tolist() == [0, 1, 128, 255, 255]


def test_quantiles_read_the_first_16_million_values():
    n = video.QUANTILE_LIMIT + 4_000_000
    d = torch.linspace(1.0, 2.0, n)
    d[::7] = 0                                            # background, left out of the near quantile only
    d[video.QUANTILE_LIMIT:] *= 100                       # past the slices: would move both quantiles
    idx = video.depth_color_index(d)
    near = d[d > 0][:video.QUANTILE_LIMIT].quantile(0.01).log()
    far = d[:video.QUANTILE_LIMIT].quantile(0.99).log()
    assert float(far) < math.log(2.0)
    x = (1 - (d.log() - near) / (far - near)).clip(0, 1)
    assert torch.equal(idx, (x * 256).long().clamp_max(255))
    assert (idx[video.QUANTILE_LIMIT:][d[video.QUANTILE_LIMIT:] > 0] == 0).all()
    assert (idx[d == 0] == 255).all()


def test_no_positive_depth_gives_black_panels_and_one_line():
    d = torch.zeros(2, 8, 8)
    assert video.depth_color_index(d) is None
    lines = []
    panels = video.depth_panels(d, log=lines.append)
    assert panels.shape == (2, 8, 8, 3) and panels.dtype == torch.uint8 and (panels == 0).all()
    assert len(lines) == 1 and "no positive depth" in lines[0]


def test_turbo_table():
    table = video.turbo_table()
    assert table.shape == (256, 3) and table.dtype == np.uint8
    # turbo runs from dark blue through green to dark red
    assert table[0, 2] > table[0, 0] and table[255, 0] > table[255, 2] and table[128, 1] > 200
    panels = video.depth_panels(torch.tensor([[[1.0, math.e ** 2]]]), log=None)
    assert panels[0, 0, 0].tolist() == table[255].tolist() and panels[0, 0, 1].tolist() == table[0].tolist()


# measured mean absolute difference of the mp4v round trip on the frames below: 2.94 (OpenCV 4.13); the bar is
# twice that, for other builds of the encoder
MP4_BAR = 6.0


def test_mp4_round_trip(tmp_path):
    import cv2
    t, h, w = 12, 72, 88
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    frames = torch.stack([torch.stack([(xx * 3 + i * 5) % 256, (yy * 3) % 256, torch.full_like(xx, 40 + 10 * i)], -1)
                          for i in range(t)]).to(torch.uint8).numpy()
    path = video.write_mp4(frames, tmp_path / "sub" / "clip.mp4")
    cap = cv2.VideoCapture(str(path))
    try:
        assert cap.isOpened()
        assert cap.get(cv2.CAP_PROP_FPS) == pytest.approx(30)
        back = []
        while True:
            ok, frame = cap.read()
            if not ok:
                break
            back.append(frame[..., ::-1])
    finally:
        cap.release()
    back = np.stack(back)
    assert back.shape == frames.shape
    mad = float(np.abs(back.astype(np.float64) - frames).mean())
    print(f"mp4v round trip: mean absolute difference {mad:.3f}")
    assert mad < MP4_BAR
    with pytest.raises(ValueError, match="uint8 frames"):
        video.write_mp4(frames.astype(np.float32), tmp_path / "bad.mp4")
    with pytest.raises(ValueError, match="uint8 frames"):
        video.write_mp4(frames[:0], tmp_path / "empty.mp4")


def test_missing_opencv_is_named(monkeypatch):
    import builtins
    real = builtins.__import__

    def no_cv2(name, *a, **k):
        if name == "cv2":
            raise ImportError("No module named 'cv2'")
        return real(name, *a, **k)

    monkeypatch.setattr(builtins, "__import__", no_cv2)
    with pytest.raises(ImportError, match="opencv-python-headless"):
        video.write_mp4(np.zeros((1, 8, 8, 3), np.uint8), "unused.mp4")


def test_render_video_arguments(tmp_path):
    from pixelsplat_b200.evaluation import __main__ as cli
    base = ["--dataset-root", "d", "--index", "i.json", "--checkpoint", "c.ckpt", "--output", str(tmp_path)]
    args = cli.parse_render_video(base)
    assert args.video == ["rgb", "wobble"] and args.preset == "re10k" and args.scene is None and args.seed is None
    args = cli.parse_render_video(base + ["--video", "interpolation_exagerrated", "rgb", "rgb", "--scene", "a",
                                          "--scene", "b", "--preset", "re10k_3_view", "--seed", "3"])
    assert args.video == ["interpolation_exagerrated", "rgb"] and args.scene == ["a", "b"] and args.seed == 3
    for bad in (["--video", "spin"], ["--video"], ["--preset", "nope"]):
        with pytest.raises(SystemExit):
            cli.parse_render_video(base + bad)
    with pytest.raises(SystemExit):
        cli.parse_render_video(base[2:])                  # no --dataset-root


def test_val_videos_argument():
    from pixelsplat_b200.training.__main__ import parse
    base = ["--dataset-root", "d", "--output", "o"]
    assert not parse(base).val_videos
    assert parse(base + ["--val-every", "5", "--val-videos"]).val_videos
    with pytest.raises(SystemExit):
        parse(base + ["--val-videos"])                    # videos are part of a validation
