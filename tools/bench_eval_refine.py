#!/usr/bin/env python
"""Times evaluation with test-time refinement per scene on the GPU, on the re10k_tiny test scenes
(tests/golden/re10k_tiny, 256 x 256) with a random-weight re10k encoder (393 216 Gaussians per scene, the real
size) and seeded LPIPS weights, for two routes:
  memory  the in-memory route: `evaluate --refine-steps N` (Evaluator with `refine`): encode, pack, refine on the
          context views, unpack, render the targets, score;
  files   the file route: `export-ply --write-frame`, then `refine-ply --steps N`, then `render-ply`.
Both routes run the commands' own functions (pixelsplat_b200.evaluation.__main__) with one encoder, decoder and LPIPS
built up front, so that neither pays for model construction or checkpoint loading; everything they write goes to a
temporary directory.  A round is one pass of a route over every scene, timed with the host clock up to a device
synchronise; the routes alternate, after one warm-up round each, and each number is the median over --rounds.
Per scene it reports the wall time of each route, the memory route's split from its Benchmarker (encoder, refine:
pack + refine + unpack, decoder: the target renders; the rest is the metrics, PNGs and data loading), and the PLY
bytes each route writes, computed from the shapes.  Prints one JSON line with the card's name and power limit, read
in the same run.

    python tools/bench_eval_refine.py [--refine-steps 100 1000] [--rounds 5]
"""
import argparse
import json
import statistics
import sys
import tempfile
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from oracle import lpips_oracle as lo  # noqa: E402
from pixelsplat_b200 import ply_export as pe  # noqa: E402
from pixelsplat_b200.evaluation import __main__ as cli  # noqa: E402
from pixelsplat_b200.evaluation import presets as ev  # noqa: E402
from pixelsplat_b200.lpips import Lpips  # noqa: E402
from tests import dataset_golden as dg  # noqa: E402
from tools.bench_depth import gpu_identity  # noqa: E402

DEV = "cuda:0"
INDEX = dg.DATA / "evaluation_index.json"
DATA = ["--dataset-root", str(dg.DATA), "--index", str(INDEX), "--num-workers", "0"]


def prebuilt_models():
    """The commands' model and LPIPS constructors replaced by one random-weight re10k encoder, its decoder and seeded
    LPIPS, built once on the device."""
    torch.manual_seed(0)
    encoder, decoder = ev.build_model("re10k", ev.dataset_cfg(dg.DATA, INDEX))
    encoder, decoder = encoder.to(DEV).eval(), decoder.to(DEV)
    lpips = Lpips()
    lpips.load_state_dict(lo.random_state_dict(0))
    lpips = lpips.to(DEV).eval()
    ev.build_model = lambda preset, cfg: (encoder, decoder)
    cli.load_preset_checkpoint = lambda path, encoder, preset: 0
    cli._lpips = lambda args, device: lpips


def timed(fn) -> float:
    torch.cuda.synchronize()
    start = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - start


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--refine-steps", type=int, nargs="+", default=[100, 1000])
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_refine: no CUDA device; the times need an H100")
    if args.rounds < 5:
        raise SystemExit("bench_eval_refine: --rounds must be at least 5")
    prebuilt_models()
    scenes = len(dg.expected("test"))
    res = {"scenes": scenes, "rounds": args.rounds}
    with tempfile.TemporaryDirectory() as tmp:
        tmp = Path(tmp)
        checkpoint = ["--checkpoint", str(tmp / "unused.ckpt"), "--preset", "re10k"]
        for steps in args.refine_steps:
            benchmarks = []

            def memory():
                cli.evaluate(DATA + checkpoint + ["--output", str(tmp / "memory"), "--refine-steps", str(steps)])
                benchmarks.append(json.loads((tmp / "memory" / "benchmark.json").read_text()))

            def files():
                cli.export_ply(DATA + checkpoint + ["--output", str(tmp / "ply"), "--write-frame"])
                cli.refine_ply(DATA + ["--ply", str(tmp / "ply"), "--output", str(tmp / "refined"),
                                       "--steps", str(steps)])
                cli.render_ply(DATA + ["--ply", str(tmp / "refined"), "--output", str(tmp / "files")])

            memory(), files()                        # warm-up
            benchmarks.clear()
            walls = {"memory": [], "files": []}
            for _ in range(args.rounds):
                walls["memory"].append(timed(memory))
                walls["files"].append(timed(files))
            key = f"steps{steps}"
            for route, ts in walls.items():
                res[f"{key}_{route}_ms_per_scene"] = statistics.median(ts) * 1e3 / scenes
                res[f"{key}_{route}_spread_ms_per_scene"] = (max(ts) - min(ts)) * 1e3 / scenes
            for tag in ("encoder", "refine", "decoder"):
                per_round = [sum(b[tag]) * 1e3 / scenes for b in benchmarks]
                res[f"{key}_memory_{tag}_ms_per_scene"] = statistics.median(per_round)
            res[f"{key}_memory_rest_ms_per_scene"] = res[f"{key}_memory_ms_per_scene"] - sum(
                res[f"{key}_memory_{tag}_ms_per_scene"] for tag in ("encoder", "refine", "decoder"))
        # the PLY bytes of one scene, from the shapes: the export and the refined copy, both written once
        layout = next(iter((tmp / "ply").glob("*.ply")))
        from pixelsplat_b200.ply_import import parse_header
        head = parse_header(layout.read_bytes()[:1 << 20])
        ply_bytes = head.body_offset + head.count * len(head.properties) * 4
        res.update(gaussians_per_scene=head.count, floats_per_record=len(head.properties),
                   files_ply_bytes_written_per_scene=2 * ply_bytes, memory_ply_bytes_written_per_scene=0)
        assert head.properties == tuple(pe.ply_properties(3))
    res.update(gpu_identity(0))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
