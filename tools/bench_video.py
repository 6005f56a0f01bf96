#!/usr/bin/env python
"""Times the videos of one 256 x 256 scene (the first test scene of tests/golden/re10k_tiny, re10k preset encoder
with seeded random weights), split into the steps `pixelsplat_b200.video.render_video` takes:
  trunk      encoder.trunk, once per scene
  tails      the probabilistic and the deterministic tail, per video
  render     the multi-view render with the fused depth channel, in chunks of 32 views, both tails
  panels     the frame pass of the colour, the depth colour map and the layout, both tails
  copy       the device-to-host copy of the laid-out frames
  encode     the loop-reverse and the mp4v encode of write_mp4 (host clock)
Device steps are CUDA events, read once the scene has finished; each number is the median over --repeats scenes.
Prints one JSON line with the card's name and power limit, read in the same run.

    python tools/bench_video.py [--videos rgb wobble] [--repeats 5] [--out FILE]
"""
import argparse
import json
import statistics
import sys
import tempfile
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from tools.bench_depth import gpu_identity  # noqa: E402

DEV = torch.device("cuda", 0)


def one_scene(encoder, decoder, batch, names, directory: Path) -> dict:
    from pixelsplat_b200 import video
    from pixelsplat_b200.encoder.encoder_tail import EncoderEpipolarTail
    from pixelsplat_b200.evaluation.frames import frame_pass
    from pixelsplat_b200.evaluation.image_io import comparison_layout
    ctx, tgt = batch["context"], batch["target"]
    event = lambda: torch.cuda.Event(enable_timing=True)
    marks, host = {}, {}
    torch.cuda.synchronize()
    with torch.no_grad():
        start = event()
        start.record()
        features, _ = encoder.trunk(ctx)
        end = event()
        end.record()
        marks["trunk"] = [(start, end)]
        for name in names:
            ext, k = (c.to(DEV).contiguous()[None] for c in video.video_trajectory(ctx, tgt, name))
            t = ext.shape[1]
            near = ctx["near"][:1, :1].expand(-1, t).contiguous()
            far = ctx["far"][:1, :1].expand(-1, t).contiguous()
            columns = []
            for deterministic in (False, True):
                e = [event() for _ in range(4)]
                e[0].record()
                g = EncoderEpipolarTail.forward(encoder, features, ctx, 0, deterministic)
                e[1].record()
                color, depth = [], []
                for i in range(0, t, video.CHUNK):
                    out = decoder.forward(g, ext[:, i:i + video.CHUNK], k[:, i:i + video.CHUNK],
                                          near[:, i:i + video.CHUNK], far[:, i:i + video.CHUNK], (256, 256),
                                          depth_mode="depth")
                    color.append(out.color[0])
                    depth.append(out.depth[0])
                e[2].record()
                columns.append((frame_pass(torch.cat(color), frames=True, planes=False).frames.permute(0, 3, 1, 2),
                                video.depth_panels(torch.cat(depth), log=None).permute(0, 3, 1, 2)))
                e[3].record()
                marks.setdefault(f"{name}/tails", []).append((e[0], e[1]))
                marks.setdefault(f"{name}/render", []).append((e[1], e[2]))
                marks.setdefault(f"{name}/panels", []).append((e[2], e[3]))
            e = [event() for _ in range(3)]
            e[0].record()
            frames = comparison_layout(*columns).permute(0, 2, 3, 1)
            e[1].record()
            frames = frames.cpu()
            e[2].record()
            marks[f"{name}/panels"].append((e[0], e[1]))
            marks[f"{name}/copy"] = [(e[1], e[2])]
            t0 = time.perf_counter()
            if video.VIDEOS[name].loop_reverse:
                frames = torch.cat([frames, frames.flip(0)[1:-1]])
            video.write_mp4(frames.numpy(), directory / f"{name}.mp4")
            host[f"{name}/encode"] = 1e3 * (time.perf_counter() - t0)
    torch.cuda.synchronize()
    out = {k: sum(a.elapsed_time(b) for a, b in v) for k, v in marks.items()}
    out.update(host)
    return out


def main() -> None:
    p = argparse.ArgumentParser()
    p.add_argument("--videos", nargs="+", default=["rgb", "wobble"])
    p.add_argument("--repeats", type=int, default=5)
    p.add_argument("--out", type=Path, default=None, help="also write the JSON line to this file")
    args = p.parse_args()
    from pixelsplat_b200.data import device_shim
    from pixelsplat_b200.evaluation import presets as ev
    data = ROOT / "tests" / "golden" / "re10k_tiny"
    torch.manual_seed(0)
    cfg = ev.dataset_cfg(data, data / "evaluation_index.json")
    encoder, decoder = ev.build_model("re10k", cfg)
    encoder, decoder = encoder.to(DEV).eval(), decoder.to(DEV)
    batch = next(iter(torch.utils.data.DataLoader(ev.make_test_dataset(cfg), batch_size=1, num_workers=0)))
    batch = encoder.get_data_shim()(device_shim(batch, (256, 256), DEV))
    runs = []
    with tempfile.TemporaryDirectory() as tmp:
        one_scene(encoder, decoder, batch, args.videos, Path(tmp))             # warm-up
        for _ in range(args.repeats):
            runs.append(one_scene(encoder, decoder, batch, args.videos, Path(tmp)))
    median = {k: round(statistics.median(r[k] for r in runs), 2) for k in runs[0]}
    line = json.dumps({"scene": batch["scene"][0], "videos": args.videos, "repeats": args.repeats,
                       "ms": median, "total_ms": round(sum(median.values()), 1), **gpu_identity(0)})
    print(line)
    if args.out is not None:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text(line + "\n")


if __name__ == "__main__":
    main()
