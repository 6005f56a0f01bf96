"""ps_view_overlap and the evaluation-index generator on the GPU, against the reference's own generator
(tests/golden/evaluation_index_v1.npz, made by oracle/make_index_golden.py): the counts on every pair the reference
evaluated, the index entry for entry, determinism, graph capture, and the command line on re10k_tiny."""
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from pixelsplat_b200.evaluation import __main__ as cli
from pixelsplat_b200.evaluation import index_generator as ig
from tests import index_util
from tests import view_overlap_f64 as vo
from tests.test_index_generator_cpu import TAU

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
GOLDEN = ROOT / "tests" / "golden" / "evaluation_index_v1.npz"
DEV = "cuda:0"


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLDEN)
    return z, json.loads(str(z["configs"])), json.loads(str(z["entries"]))


def _cams(z, family):
    return (torch.from_numpy(z[f"cam/{family}/extrinsics"]).to(DEV),
            torch.from_numpy(z[f"cam/{family}/intrinsics"]).to(DEV))


def test_counts_equal_the_reference_outside_flagged_rays(golden):
    """Every recorded (context, k) pair: the kernel's two counts equal overlap * h * w of the reference, except by at
    most the rays the float64 restatement flags within TAU of a decision (or the pair's masks within MASK_TOL)."""
    z, configs, _ = golden
    pairs = diffs = 0
    worst = 0.0
    for config, c in configs.items():
        for family in index_util.FAMILIES:
            rec = z[f"{config}/{family}/pairs"]
            if not len(rec):
                continue
            E, K = _cams(z, family)
            for ctx in np.unique(rec[:, 0]):
                sel = rec[rec[:, 0] == ctx]
                first, last = int(sel[:, 1].min()), int(sel[:, 1].max())
                got = ig.view_overlap_counts(E, K, c["h"], c["w"], int(ctx), first, last - first + 1).cpu().numpy()
                for _, k, ca, cb in sel:
                    pairs += 1
                    g = got[k - first]
                    if (g[0], g[1]) == (ca, cb):
                        continue
                    _, flagged = vo.pair_counts(z[f"cam/{family}/extrinsics"], z[f"cam/{family}/intrinsics"], c["h"],
                                                c["w"], int(ctx), int(k), TAU)
                    for x, want, f in zip(g, (ca, cb), flagged):
                        d = abs(int(x) - int(want))
                        assert d <= f, (config, family, int(ctx), int(k), int(x), int(want), f)
                        if d:
                            diffs += 1
                            worst = max(worst, d / f)
    print(f"{pairs} pairs, {diffs} directions differ from the reference, worst use of the flagged rays {worst:.3f}")


def _entries(z, config, c):
    cfg = ig.EvaluationIndexGeneratorCfg(**c["cfg"])
    g = torch.Generator()
    g.manual_seed(cfg.seed)
    out = {}
    for family in index_util.FAMILIES:
        e = ig.generate_scene_entry(*_cams(z, family), c["h"], c["w"], cfg, g)
        out[family] = None if e is None else {"context": list(e.context), "target": list(e.target)}
    return out


@pytest.mark.parametrize("config", [c[0] for c in index_util.CONFIGS])
def test_index_equals_the_reference(golden, config):
    z, configs, entries = golden
    assert _entries(z, config, configs[config]) == entries[config]


def test_two_runs_write_identical_bytes(golden, tmp_path):
    z, configs, _ = golden
    texts = []
    for run in range(2):
        index = _entries(z, "default", configs["default"])
        from pixelsplat_b200.data.view_sampler import IndexEntry
        index = {k: None if v is None else IndexEntry(tuple(v["context"]), tuple(v["target"])) for k, v in index.items()}
        (path,) = ig.save_index(index, tmp_path / str(run))
        texts.append(path.read_bytes())
    assert texts[0] == texts[1]


def test_counts_repeat_and_replay_in_a_cuda_graph(golden):
    """The launch is graph-capturable (no host synchronisation inside), and repeats and replays give the same
    counts: the CTA counts are integers added atomically."""
    z, _, _ = golden
    E, K = _cams(z, "rotate")
    ref = ig.view_overlap_counts(E, K, 256, 256, 150, 14, 273).clone()
    assert torch.equal(ig.view_overlap_counts(E, K, 256, 256, 150, 14, 273), ref)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ig.view_overlap_counts(E, K, 256, 256, 150, 14, 273)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ig.view_overlap_counts(E, K, 256, 256, 150, 14, 273)
    for _ in range(3):
        out.fill_(-1)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, ref)


@pytest.mark.parametrize("workers", [0, 8])
def test_command_line_on_re10k_tiny(golden, tmp_path, workers):
    """generate-index on re10k_tiny in the small configuration writes the index the reference's generator wrote
    from the same chunk (with 8 workers; one chunk gives every worker count the same order), and --video its
    video index."""
    z, _, _ = golden
    out = tmp_path / "index"
    cli.main(["generate-index", "--dataset-root", str(ROOT / "tests" / "golden" / "re10k_tiny"), "--output", str(out),
              "--min-distance", "2", "--max-distance", "6", "--num-workers", str(workers), "--video"])
    assert (out / "evaluation_index.json").read_text() == str(z["re10k_tiny"])
    video = json.loads((out / "evaluation_index_video.json").read_text())
    for scene, entry in json.loads(str(z["re10k_tiny"])).items():
        a, b = entry["context"]
        assert video[scene] == {"context": [a, b], "target": list(range(a, b + 1))}
