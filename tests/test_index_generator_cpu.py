"""The evaluation-index generator's host side (pixelsplat_b200/evaluation/index_generator.py) without a GPU: the walk
replayed on the overlaps the reference's own generator recorded (tests/golden/evaluation_index_v1.npz, made by
oracle/make_index_golden.py), its float32 thresholds, the JSON files, the command line, the camera-only reader, the
ABI's refusals, and the float64 restatement of the kernel against the reference's counts."""
import ctypes
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from pixelsplat_b200.data import DatasetRE10k
from pixelsplat_b200.evaluation import __main__ as cli
from pixelsplat_b200.evaluation import index_generator as ig
from pixelsplat_b200.evaluation.presets import dataset_cfg
from tests import index_util
from tests import view_overlap_f64 as vo

ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden" / "evaluation_index_v1.npz"
TINY = ROOT / "tests" / "golden" / "re10k_tiny"


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLDEN)
    return z, json.loads(str(z["configs"])), json.loads(str(z["entries"]))


def _cfg(fields: dict) -> ig.EvaluationIndexGeneratorCfg:
    return ig.EvaluationIndexGeneratorCfg(**fields)


class _Recorded:
    """The counts of one candidate range, served from the reference's records; reading a frame it never evaluated
    fails, and every frame read is logged."""

    def __init__(self, pairs: dict, context: int, first: int, log: list):
        self.pairs, self.context, self.first, self.log = pairs, context, first, log

    def __getitem__(self, i: int):
        k = self.first + i
        assert (self.context, k) in self.pairs, f"the walk read frame {k} from {self.context}, which the reference " \
                                                f"did not evaluate"
        self.log.append((self.context, k))
        return self.pairs[(self.context, k)]


@pytest.mark.parametrize("config", [c[0] for c in index_util.CONFIGS])
def test_walk_replays_the_reference(golden, config):
    """Fed the reference's overlaps, the walk evaluates the same pairs in the same order and draws the same entries,
    with one generator across the scenes."""
    z, configs, entries = golden
    c = configs[config]
    cfg = _cfg(c["cfg"])
    generator = torch.Generator()
    generator.manual_seed(cfg.seed)
    for family in index_util.FAMILIES:
        rec = z[f"{config}/{family}/pairs"]
        pairs = {(int(a), int(b)): (int(x), int(y)) for a, b, x, y in rec}
        log: list = []
        v = z[f"cam/{family}/extrinsics"].shape[0]
        entry = ig.scene_entry(v, c["h"], c["w"], cfg, generator,
                               lambda ctx, first, count: _Recorded(pairs, ctx, first, log))
        assert log == [(int(a), int(b)) for a, b, _, _ in rec], family
        got = None if entry is None else {"context": list(entry.context), "target": list(entry.target)}
        assert got == entries[config][family], family


def test_candidate_range_covers_both_walks():
    cfg = ig.EvaluationIndexGeneratorCfg()
    assert ig.candidate_range(150, 300, cfg) == (14, 273)        # 150 -+ 136
    assert ig.candidate_range(0, 300, cfg) == (45, 92)           # only the forward walk: 45 .. 136
    assert ig.candidate_range(299, 300, cfg) == (163, 92)
    assert ig.candidate_range(10, 40, cfg) is None               # shorter than min_distance on both sides
    far = ig.EvaluationIndexGeneratorCfg(num_target_views=1, min_distance=10, max_distance=3)
    assert ig.candidate_range(20, 40, far) == (10, 21)           # the walk still evaluates c +- min_distance


def test_overlap_thresholds_are_float32():
    """The reference compares a 0-d float32 tensor with Python floats: torch rounds the float to float32.  Checked
    against torch itself, with overlaps equal to float32(0.6) and thresholds that round either way."""
    f32 = np.float32
    lo = [0.6, float(np.nextafter(f32(0.6), f32(1))), float(f32(0.6)) + 1e-9, float(f32(0.6)) - 1e-9, 0.599999999]
    overlaps = [f32(3) / f32(5), np.nextafter(f32(0.6), f32(0)), np.nextafter(f32(0.6), f32(1)), f32(1), f32(0)]
    assert f32(3) / f32(5) == f32(0.6)
    for a in lo:
        for hi in (1.0, float(f32(0.6)), 0.6000000001):
            cfg = ig.EvaluationIndexGeneratorCfg(min_overlap=a, max_overlap=hi)
            for x in overlaps:
                t = torch.tensor(x, dtype=torch.float32)
                assert ig.in_overlap_range(x, cfg) == bool(a <= t <= hi), (a, hi, x)
    # a walk at h * w = 5 with 3 of 5 rays overlapping both ways sits exactly on min_overlap = 0.6: a candidate
    cfg = ig.EvaluationIndexGeneratorCfg(num_target_views=1, min_distance=1, max_distance=1)
    g = torch.Generator().manual_seed(0)
    counts = np.array([[5, 5], [3, 3], [0, 0]])
    assert ig.walk_context(0, 3, counts, 0, 5, cfg, g) is not None
    counts[1] = (2, 3)
    assert ig.walk_context(0, 3, counts, 0, 5, cfg, g) is None


def test_json_layout_and_video_index(tmp_path):
    from pixelsplat_b200.data.view_sampler import IndexEntry
    index = {"a": IndexEntry((3, 9), (4, 5, 8)), "b": None, "c": IndexEntry((0, 2), (0, 1, 2))}
    main, video = ig.save_index(index, tmp_path / "out", video=True)
    assert main.read_text() == ('{"a": {"context": [3, 9], "target": [4, 5, 8]}, "b": null, '
                                '"c": {"context": [0, 2], "target": [0, 1, 2]}}')
    assert json.loads(video.read_text()) == {"a": {"context": [3, 9], "target": list(range(3, 10))}, "b": None,
                                             "c": {"context": [0, 2], "target": [0, 1, 2]}}
    assert video.name == "evaluation_index_video.json"
    assert ig.save_index(index, tmp_path / "plain") == [tmp_path / "plain" / "evaluation_index.json"]


def test_command_line_parsing(capsys):
    a = cli.parse_generate_index(["--dataset-root", "d", "--output", "o"])
    assert a.cfg == ig.EvaluationIndexGeneratorCfg(output_path=Path("o"))
    assert a.num_workers == 8 and not a.video
    a = cli.parse_generate_index(["--dataset-root", "d", "--output", "o", "--num-target-views", "2", "--min-overlap",
                                  "0.5", "--max-overlap", "0.9", "--min-distance", "2", "--max-distance", "6",
                                  "--seed", "7", "--num-workers", "0", "--video"])
    assert a.cfg == ig.EvaluationIndexGeneratorCfg(2, 2, 6, 0.5, 0.9, Path("o"), 7) and a.num_workers == 0 and a.video
    for bad in (["--min-distance", "1"], ["--num-workers", "-1"], ["--max-distance", "-2"]):
        with pytest.raises(SystemExit):
            cli.parse_generate_index(["--dataset-root", "d", "--output", "o", *bad])
    with pytest.raises(SystemExit):
        cli.parse_generate_index(["--help"])
    assert "depends on it" in capsys.readouterr().out


class _AllViews:
    """The reference's `all` view sampler: every frame is a context and a target view."""

    def sample(self, scene, extrinsics, intrinsics):
        frames = torch.arange(extrinsics.shape[0])
        return frames, frames


@pytest.mark.parametrize("workers", [0, 8])
def test_camera_reader_matches_the_full_reader(workers):
    """On re10k_tiny the camera-only reader yields the scenes, order and cameras the full reader yields with the `all`
    sampler, and skips the same ones, through the same DataLoader."""
    cfg = dataset_cfg(TINY, TINY / "evaluation_index.json")
    full = torch.utils.data.DataLoader(DatasetRE10k(cfg, "test", _AllViews()), batch_size=1, num_workers=workers)
    cams = ig.camera_loader(TINY, workers)
    a, b = list(full), list(cams)
    assert [x["scene"] for x in a] == [x["scene"] for x in b] == [["aaa"], ["bbb"], ["eee"], ["fff"]]
    for x, y in zip(a, b):
        assert torch.equal(x["target"]["extrinsics"], y["extrinsics"])
        assert torch.equal(x["target"]["intrinsics"], y["intrinsics"])
        assert int(y["num_frames"]) == x["target"]["extrinsics"].shape[1]


def test_camera_reader_skips_missing_and_misshapen_images(tmp_path):
    chunk = torch.load(TINY / "test" / "000000.torch", weights_only=True)
    cfg = dataset_cfg(TINY, TINY / "evaluation_index.json")
    ds = DatasetRE10k(cfg, "test", None, cameras_only=True)
    ok = ds.convert_example(chunk[0])
    assert ok is not None and ok["num_frames"] == len(chunk[0]["images"])
    assert ds.convert_example({**chunk[0], "images": chunk[0]["images"][:-1]}) is None
    from io import BytesIO

    from PIL import Image
    buf = BytesIO()
    Image.new("RGB", (640, 352)).save(buf, format="JPEG")
    small = torch.frombuffer(bytearray(buf.getvalue()), dtype=torch.uint8)
    assert ds.convert_example({**chunk[0], "images": [small] + list(chunk[0]["images"][1:])}) is None


ABI_CHILD = """
import ctypes, json, sys
from pixelsplat_b200 import _lib
FAKE = ctypes.c_void_p(0x1000)
out = []
for v, h, w, null, c, first, count in json.loads(sys.argv[1]):
    e, k, o = [None if n == null else FAKE for n in ("extrinsics", "intrinsics", "counts")]
    rc = _lib.lib.ps_view_overlap(v, h, w, e, k, c, first, count, o, None)
    out.append([rc, _lib.lib.ps_last_error().decode()])
print(json.dumps(out))
"""
# (views, grid_h, grid_w, NULL pointer, context, first, count) -> expected return code
ABI_CASES = {**{(10, 4, 4, p, 0, 1, 3): 1 for p in ("extrinsics", "intrinsics", "counts")},
             (0, 4, 4, None, 0, 0, 1): 1, (10, 0, 4, None, 0, 1, 3): 1, (10, 4, 0, None, 0, 1, 3): 1,
             (10, 4, 4, None, 0, 1, 0): 1, (10, 4, 4, None, -1, 1, 3): 1, (10, 4, 4, None, 10, 1, 3): 1,
             (10, 4, 4, None, 0, -1, 3): 1, (10, 4, 4, None, 0, 8, 3): 1, (10, 4, 4, None, 0, 10, 1): 1,
             (70000, 4, 4, None, 0, 0, 65536): 3, (10, 65536, 32768, None, 0, 1, 3): 3,
             (10, 46341, 46341, None, 0, 1, 3): 3}


def test_abi_refuses_before_enqueuing():
    """ps_view_overlap refuses bad counts, NULL pointers and ranges outside [0, views) with PS_ERR_INVALID_ARGUMENT
    (1), and a grid it cannot launch with PS_ERR_UNSUPPORTED (3), in a child process that sees no GPU: a check that
    stopped refusing would fail there instead of launching on the fake addresses."""
    cases = list(ABI_CASES)
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-c", ABI_CHILD, json.dumps(cases)], cwd=str(ROOT), env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    for case, (rc, err) in zip(cases, json.loads(r.stdout.strip().splitlines()[-1])):
        assert rc == ABI_CASES[case], (case, rc, err)


def test_restatement_matches_the_reference_counts(golden):
    """The float64 restatement gives the reference's counts on the small configuration's pairs and on the first two
    pairs of each family at 256 x 256, within its flagged rays (TAU)."""
    z, configs, _ = golden
    for config, limit in (("small", None), ("default", 2)):
        c = configs[config]
        for family in index_util.FAMILIES:
            E, K = z[f"cam/{family}/extrinsics"], z[f"cam/{family}/intrinsics"]
            for ctx, k, ca, cb in z[f"{config}/{family}/pairs"][:limit]:
                counts, flagged = vo.pair_counts(E, K, c["h"], c["w"], int(ctx), int(k), TAU)
                for got, want, f in zip(counts, (ca, cb), flagged):
                    assert abs(got - want) <= f, (config, family, ctx, k, got, want, f)


TAU = 1e-5     # relative distance from a decision within which a ray may go either way (float32 vs float64)
