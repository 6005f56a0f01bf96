"""Evaluation with test-time refinement on the GPU (evaluate --refine-steps, Evaluator(refine=...),
ply_refine.refine_gaussians), on re10k_tiny with a random-weight checkpoint and seeded LPIPS:
  1. the in-memory route equals the file route (export-ply --write-frame, refine-ply, render-ply) bit for bit:
     target PNGs, per-scene metrics and refine.json, with the MSE loss, with L1 + D-SSIM, position-rate decay and
     densification, and with zero steps (against render-ply of the unrefined export);
  2. refinement off is the evaluator as it was: no pack, no refinement, the same frames and metrics, no "refine"
     timings;
  3. refinement lowers each scene's context MSE and changes the frames;
  4. the three-view model is refined on its three context views;
  5. two in-memory runs give the same bits;
  6. the export frame's centre is torch.median's, computed in deterministic mode too.
Identity and repeatability need torch's deterministic mode (the rasterizer's fixed-order backward); the fixture sets
it and restores it."""
import contextlib
import json

import pytest
import torch

from pixelsplat_b200 import ply_export as pe
from pixelsplat_b200 import ply_refine as pr
from pixelsplat_b200.evaluation import __main__ as cli
from pixelsplat_b200.evaluation import presets as ev
from pixelsplat_b200.evaluation.checkpoint import save_checkpoint
from tests import dataset_golden as dg
from tests.test_evaluation_gpu import _seeded_lpips

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
INDEX = dg.DATA / "evaluation_index.json"
DATA = ["--dataset-root", str(dg.DATA), "--index", str(INDEX), "--num-workers", "0"]
CASES = {
    "mse": ("20", []),
    "dssim_densify": ("20", ["--loss", "l1-dssim", "--lr-xyz-final", "1.6e-6", "--densify-from", "5",
                             "--densify-until", "15", "--densify-every", "5", "--densify-grad", "2e-6"]),
    "zero": ("0", []),
}


@contextlib.contextmanager
def _deterministic(mp: pytest.MonkeyPatch):
    mp.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(old)


def _checkpoint(path, preset: str = "re10k"):
    torch.manual_seed(0)
    encoder, _ = ev.build_model(preset, ev.dataset_cfg(dg.DATA, INDEX, preset=preset))
    return str(save_checkpoint(path, encoder, 0))


def _evaluate(ckpt, out, *extra, preset="re10k"):
    return cli.evaluate(DATA + ["--checkpoint", ckpt, "--preset", preset, "--output", str(out), *extra])


def _frames(root) -> dict:
    """{scene/color/name.png: bytes} of every target frame under `root`."""
    return {str(p.relative_to(root)): p.read_bytes() for p in sorted(root.glob("*/color/*.png"))}


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    """Each case's in-memory route and file route, from one export; and the MSE case's in-memory route again."""
    root = tmp_path_factory.mktemp("eval_refine")
    with pytest.MonkeyPatch.context() as mp, _deterministic(mp):
        mp.setattr(cli, "_lpips", lambda args, device: _seeded_lpips())
        ckpt = _checkpoint(root / "random.ckpt")
        cli.main(["export-ply"] + DATA + ["--checkpoint", ckpt, "--preset", "re10k", "--output", str(root / "ply"),
                                          "--write-frame"])
        out = {}
        for name, (steps, extra) in CASES.items():
            memory = _evaluate(ckpt, root / name / "memory", "--refine-steps", steps, *extra)
            cli.main(["refine-ply"] + DATA + ["--ply", str(root / "ply"), "--output", str(root / name / "refined"),
                                              "--steps", steps] + extra)
            source = root / "ply" if steps == "0" else root / name / "refined"
            files = cli.render_ply(["--ply", str(source), "--output", str(root / name / "files")] + DATA)
            out[name] = memory, files
        again = _evaluate(ckpt, root / "again", "--refine-steps", CASES["mse"][0])
    return root, out, again


@pytest.mark.parametrize("case", list(CASES))
def test_in_memory_route_equals_the_file_route(runs, case):
    root, out, _ = runs
    memory, files = out[case]
    scenes = [w["scene"] for w in dg.expected("test")]
    assert sorted(memory["scenes"]) == sorted(scenes)
    a, b = _frames(root / case / "memory"), _frames(root / case / "files")
    assert len(a) == sum(len(w["target"]["index"]) for w in dg.expected("test"))
    assert a.keys() == b.keys()
    assert [k for k in a if a[k] != b[k]] == []
    assert memory["scenes"] == files["scenes"] and memory["mean"] == files["mean"]
    report = json.loads((root / case / "memory" / "refine.json").read_text())
    assert report == json.loads((root / case / "refined" / "refine.json").read_text())
    for s, r in report["scenes"].items():
        print(f"EVAL_REFINE {case} {s}: " + cli._refine_line(s, r) + f"; psnr {memory['scenes'][s]['psnr']:.4f}")
    bench = json.loads((root / case / "memory" / "benchmark.json").read_text())
    assert len(bench["refine"]) == len(scenes) and len(bench["encoder"]) == len(scenes)
    if case == "dssim_densify":
        assert any(r["gaussians_after"] != r["gaussians_before"] for r in report["scenes"].values())
        assert all("loss_after" in r for r in report["scenes"].values())
    if case == "zero":
        assert all(r["mse_before"] == r["mse_after"] for r in report["scenes"].values())


def test_refinement_lowers_the_context_mse_and_changes_the_frames(runs):
    root, _, _ = runs
    report = json.loads((root / "mse" / "memory" / "refine.json").read_text())
    assert report["steps"] == 20
    assert all(r["mse_after"] < r["mse_before"] for r in report["scenes"].values())
    refined, zero = _frames(root / "mse" / "memory"), _frames(root / "zero" / "memory")
    assert refined.keys() == zero.keys() and all(refined[k] != zero[k] for k in refined)


def test_two_in_memory_runs_give_the_same_bits(runs):
    root, out, again = runs
    assert _frames(root / "again") == _frames(root / "mse" / "memory")
    assert again == out["mse"][0]
    assert (root / "again" / "refine.json").read_bytes() == (root / "mse" / "memory" / "refine.json").read_bytes()


def test_refinement_off_is_the_evaluator_as_it_was(tmp_path, monkeypatch):
    from pixelsplat_b200.evaluation import Evaluator
    monkeypatch.setattr(cli, "_lpips", lambda args, device: _seeded_lpips())
    calls = []
    for module, name in ((pe, "pack_viewer"), (pr, "refine_records")):
        real = getattr(module, name)
        monkeypatch.setattr(module, name, lambda *a, _real=real, _name=name, **k: calls.append(_name) or _real(*a, **k))
    ckpt = _checkpoint(tmp_path / "random.ckpt")
    args = cli.parse_evaluate(DATA + ["--checkpoint", ckpt])
    cfg, loader = cli._loader(args, "re10k")
    encoder, decoder = ev.build_model("re10k", cfg)
    cli.load_preset_checkpoint(args.checkpoint, encoder, "re10k")
    plain = Evaluator(encoder.to(DEV).eval(), decoder.to(DEV), tmp_path / "plain", _seeded_lpips())
    with _deterministic(monkeypatch):
        off = _evaluate(ckpt, tmp_path / "off")
        result = plain.run(loader, seed=ev.SEED, device=DEV, log=None)
    assert calls == []
    assert not (tmp_path / "off" / "refine.json").exists()
    assert "refine" not in json.loads((tmp_path / "off" / "benchmark.json").read_text())
    assert off == {"mean": result.mean, "scenes": {s.scene: s.metrics for s in result.scenes}}
    assert all(s.refine is None for s in result.scenes)
    assert _frames(tmp_path / "off") == _frames(tmp_path / "plain")
    assert sorted(json.loads((tmp_path / "off" / "benchmark.json").read_text())) == ["decoder", "encoder"]


def test_export_centre_is_torchs_median_and_runs_in_deterministic_mode(monkeypatch):
    g = torch.Generator(device=DEV).manual_seed(3)
    for n in (1, 2, 1001, 393_216):
        means = torch.randn((n, 3), device=DEV, generator=g)
        means[::5] = means[0].clone()
        want = means.median(dim=0).values
        with _deterministic(monkeypatch):
            center, _ = pe.normalisation(means)
        assert torch.equal(center, want), n


def test_three_view_model_refines_on_its_three_context_views(tmp_path, monkeypatch):
    monkeypatch.setattr(cli, "_lpips", lambda args, device: _seeded_lpips())
    views = []
    real = pr.refine_records

    def spy(records, properties, sh_degree, **k):
        views.append((k["images"].shape[0], k["extrinsics"].shape[0], k["intrinsics"].shape[0], k["near"].shape[0]))
        return real(records, properties, sh_degree, **k)
    monkeypatch.setattr(pr, "refine_records", spy)
    ckpt = _checkpoint(tmp_path / "random.ckpt", "re10k_3_view")
    out = _evaluate(ckpt, tmp_path / "three", "--refine-steps", "5", preset="re10k_3_view")
    assert len(out["scenes"]) > 0 and views == [(3, 3, 3, 3)] * len(out["scenes"])
    report = json.loads((tmp_path / "three" / "refine.json").read_text())
    assert sorted(report["scenes"]) == sorted(out["scenes"])
    assert all(r["steps"] == 5 for r in report["scenes"].values())
