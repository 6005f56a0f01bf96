"""CPU tests of evaluation with test-time refinement (Evaluator(refine=...), evaluate --refine-steps,
ply_refine.refine_gaussians): the evaluate parser without the new flags, the refusals of refinement options without
--refine-steps, refine-ply's parser kept as it was, and refine_gaussians' refusals before any launch."""
import contextlib
import hashlib
import io
from pathlib import PosixPath

import pytest
import torch

from pixelsplat_b200 import ply_refine as pr
from pixelsplat_b200.decoder import Gaussians
from pixelsplat_b200.evaluation import __main__ as cli

EVALUATE = ["--dataset-root", "d", "--index", "i", "--checkpoint", "c"]
REFINE_PLY = ["--ply", "p", "--dataset-root", "d", "--index", "i", "--output", "o"]

# evaluate's namespaces before refinement existed
EVALUATE_NAMESPACES = [
    ([], {"dataset_root": PosixPath("d"), "index": PosixPath("i"), "seed": None, "num_workers": 4, "lpips_vgg": None,
          "lpips_lin": None, "checkpoint": PosixPath("c"), "preset": "re10k", "output": None, "deterministic": False,
          "no_frames": False, "global_step": 0}),
    (["--preset", "re10k_3_view", "--output", "o", "--deterministic", "--no-frames", "--global-step", "3", "--seed",
      "5", "--num-workers", "0", "--lpips-vgg", "v", "--lpips-lin", "l"],
     {"dataset_root": PosixPath("d"), "index": PosixPath("i"), "seed": 5, "num_workers": 0,
      "lpips_vgg": PosixPath("v"), "lpips_lin": PosixPath("l"), "checkpoint": PosixPath("c"), "preset": "re10k_3_view",
      "output": PosixPath("o"), "deterministic": True, "no_frames": True, "global_step": 3}),
]

# refine-ply's namespace before the refinement options were shared with evaluate: the defaults, then per argument
# list the entries it changes
LR = {"xyz": 0.00016, "f_dc": 0.0025, "f_rest": 0.000125, "opacity": 0.05, "scale": 0.005, "rot": 0.001}
REFINE_PLY_DEFAULTS = {
    "ply": PosixPath("p"), "dataset_root": PosixPath("d"), "index": PosixPath("i"), "output": PosixPath("o"),
    "scene": None, "steps": 100, "num_workers": 4, "lr_xyz": 0.00016, "lr_f_dc": 0.0025, "lr_f_rest": 0.000125,
    "lr_opacity": 0.05, "lr_scale": 0.005, "lr_rot": 0.001, "densify_until": 0, "densify_from": 500,
    "densify_every": 100, "densify_grad": 0.0002, "min_opacity": 0.005, "opacity_reset_every": 3000,
    "densify_seed": 0, "loss": "mse", "lambda_dssim": 0.2, "lr_xyz_final": None, "lr_xyz_steps": None, "lr": LR,
    "densify": None}
REFINE_PLY_NAMESPACES = [
    ([], {}),
    (["--steps", "0", "--scene", "a", "--scene", "b", "--lr-xyz", "1e-3", "--lr-f-rest", "0", "--num-workers", "2"],
     {"scene": ["a", "b"], "steps": 0, "num_workers": 2, "lr_xyz": 0.001, "lr_f_rest": 0.0,
      "lr": dict(LR, xyz=0.001, f_rest=0.0)}),
    (["--densify-until", "800", "--densify-from", "100", "--densify-every", "50", "--densify-grad", "1e-5",
      "--min-opacity", "0.01", "--opacity-reset-every", "0", "--densify-seed", "3"],
     {"densify_until": 800, "densify_from": 100, "densify_every": 50, "densify_grad": 1e-05, "min_opacity": 0.01,
      "opacity_reset_every": 0, "densify_seed": 3,
      "densify": pr.DensifyConfig(from_step=100, until_step=800, every=50, grad_threshold=1e-05, percent_dense=0.01,
                                  min_opacity=0.01, opacity_reset_every=0, extent=1.0, seed=3)}),
    (["--loss", "l1-dssim", "--lambda-dssim", "0.5", "--lr-xyz-final", "1.6e-6", "--lr-xyz-steps", "30"],
     {"loss": "l1_dssim", "lambda_dssim": 0.5, "lr_xyz_final": 1.6e-06, "lr_xyz_steps": 30}),
    (["--steps", "20", "--lr-xyz-final", "1e-6", "--lr-rot=0.5", "--densify-unt", "3"],
     {"steps": 20, "lr_rot": 0.5, "densify_until": 3, "lr_xyz_final": 1e-06, "lr": dict(LR, rot=0.5),
      "densify": pr.DensifyConfig(until_step=3)}),
]
# sha256 and length of `refine-ply --help` at 80 columns before the options were shared
REFINE_PLY_HELP = ("eb405a3d386830f27df3645901a41df9224c57d2af35ab34ea9d87cd8c2bfa5e", 5190)

REFINE_OPTIONS = [["--lr-xyz", "1e-3"], ["--lr-f-dc", "0"], ["--lr-f-rest", "0"], ["--lr-opacity", "0"],
                  ["--lr-scale", "0"], ["--lr-rot", "0"], ["--densify-until", "10"], ["--densify-from", "1"],
                  ["--densify-every", "2"], ["--densify-grad", "1e-5"], ["--min-opacity", "0.1"],
                  ["--opacity-reset-every", "0"], ["--densify-seed", "1"], ["--loss", "l1-dssim"],
                  ["--lambda-dssim", "0.5"], ["--lr-xyz-final", "1e-6"], ["--lr-xyz-steps", "9"]]


@pytest.mark.parametrize("extra,want", EVALUATE_NAMESPACES)
def test_evaluate_without_refinement_parses_as_before(extra, want):
    args = cli.parse_evaluate(EVALUATE + extra)
    assert list(vars(args).items()) == list({**want, "refine": None}.items())


def test_evaluate_with_refinement_collects_the_options():
    args = cli.parse_evaluate(EVALUATE + ["--refine-steps", "0"])
    assert args.refine == dict(steps=0, lr=LR, densify=None, loss="mse", lambda_dssim=0.2, lr_xyz_final=None,
                               lr_xyz_steps=None)
    args = cli.parse_evaluate(EVALUATE + ["--refine-steps", "20", "--loss", "l1-dssim", "--lr-xyz-final", "1.6e-6",
                                          "--densify-from", "5", "--densify-until", "15", "--densify-every", "5",
                                          "--densify-grad", "2e-6", "--lr-rot", "0.5"])
    assert args.refine == dict(steps=20, lr=dict(LR, rot=0.5),
                               densify=pr.DensifyConfig(from_step=5, until_step=15, every=5, grad_threshold=2e-6),
                               loss="l1_dssim", lambda_dssim=0.2, lr_xyz_final=1.6e-6, lr_xyz_steps=None)
    # the evaluator's keys and nothing else: the options live in `refine`
    assert set(vars(args)) == set(EVALUATE_NAMESPACES[0][1]) | {"refine"}
    pr.check_refine_options(**args.refine)


@pytest.mark.parametrize("option", REFINE_OPTIONS, ids=lambda o: o[0])
def test_evaluate_refuses_a_refinement_option_without_refine_steps(option, capsys):
    with pytest.raises(SystemExit) as e:
        cli.parse_evaluate(EVALUATE + option)
    assert e.value.code == 2
    assert f"{option[0]} without --refine-steps" in capsys.readouterr().err
    cli.parse_evaluate(EVALUATE + option + ["--refine-steps", "1"] +
                       (["--lr-xyz-final", "1e-6"] if option[0] == "--lr-xyz-steps" else []))


def test_evaluate_refuses_abbreviated_and_joined_options_and_negative_steps(capsys):
    for extra in (["--lambda", "0.5"], ["--lr-rot=0.5"], ["--densify-unt", "3"]):
        with pytest.raises(SystemExit):
            cli.parse_evaluate(EVALUATE + extra)
        assert "without --refine-steps" in capsys.readouterr().err
    for bad in (["--refine-steps", "-1"], ["--refine-steps", "1.5"],
                ["--refine-steps", "5", "--lr-xyz-steps", "3"],
                ["--refine-steps", "5", "--densify-until", "10", "--densify-every", "0"]):
        with pytest.raises(SystemExit):
            cli.parse_evaluate(EVALUATE + bad)


@pytest.mark.parametrize("extra,changes", REFINE_PLY_NAMESPACES)
def test_refine_ply_namespace_is_unchanged(extra, changes):
    args = cli.parse_refine_ply(REFINE_PLY + extra)
    assert list(vars(args).items()) == list({**REFINE_PLY_DEFAULTS, **changes}.items())


def test_refine_ply_help_is_unchanged(monkeypatch):
    monkeypatch.setenv("COLUMNS", "80")
    out = io.StringIO()
    with contextlib.redirect_stdout(out), pytest.raises(SystemExit):
        cli.parse_refine_ply(["--help"])
    text = out.getvalue().encode()
    assert (hashlib.sha256(text).hexdigest(), len(text)) == REFINE_PLY_HELP


def test_evaluate_help_names_the_steps_flag_of_the_decay(monkeypatch):
    monkeypatch.setenv("COLUMNS", "200")
    out = io.StringIO()
    with contextlib.redirect_stdout(out), pytest.raises(SystemExit):
        cli.parse_evaluate(["--help"])
    assert "(default: --refine-steps; 3DGS: 30000)" in out.getvalue()


def _scene(batch: int) -> Gaussians:
    n = 5
    return Gaussians(torch.zeros(batch, n, 3), torch.eye(3).expand(batch, n, 3, 3).contiguous(),
                     torch.zeros(batch, n, 3, 25), torch.full((batch, n), 0.5))


def _views():
    return dict(context_extrinsics=torch.eye(4)[None].expand(2, 4, 4), intrinsics=torch.eye(3)[None].expand(2, 3, 3),
                near=torch.ones(2), far=torch.full((2,), 100.0), images=torch.zeros(2, 3, 8, 8),
                background_color=torch.zeros(3))


@pytest.mark.parametrize("batch,steps,options,match", [
    (1, -1, {}, "`steps` must be an int >= 0"),
    (1, 1.5, {}, "`steps` must be an int >= 0"),
    (2, 3, {}, "batch dimension of 1"),
    (1, 3, {"loss": "l2"}, "`loss` must be one of"),
    (1, 3, {"lr": {"xyzw": 1.0}}, "unknown learning-rate group"),
    (1, 3, {"densify": {"until_step": 3}}, "`densify` must be a DensifyConfig"),
    (1, 3, {"lambda_dssim": 2.0}, "`lambda_dssim` must be a number in"),
    (1, 3, {"lr_xyz_steps": 3}, "`lr_xyz_steps` needs `lr_xyz_final`"),
    (1, 3, {"sh_degree": 2}, "unknown option sh_degree"),
])
def test_refine_gaussians_refuses_before_any_launch(monkeypatch, batch, steps, options, match):
    from pixelsplat_b200 import ply_export, ply_import

    def launched(*a, **k):
        raise AssertionError("a kernel was launched before the arguments were checked")
    for module, name in ((ply_export, "pack_viewer"), (pr, "refine_records"), (ply_import, "unpack_records")):
        monkeypatch.setattr(module, name, launched)
    with pytest.raises(ValueError, match=match):
        pr.refine_gaussians(_scene(batch), torch.eye(4), steps=steps, **_views(), **options)


def test_evaluator_refuses_bad_refinement_settings():
    from pixelsplat_b200.evaluation import Evaluator

    class Encoder(torch.nn.Module):
        def get_data_shim(self):
            return lambda batch: batch
    for refine, match in (({}, "must hold 'steps'"), ({"steps": -1}, "`steps` must be an int >= 0"),
                          ({"steps": 2, "densify_until": 3}, "unknown option densify_until")):
        with pytest.raises(ValueError, match=match):
            Evaluator(Encoder(), torch.nn.Module(), refine=refine)
    assert Evaluator(Encoder(), torch.nn.Module()).refine is None
    assert Evaluator(Encoder(), torch.nn.Module(), refine={"steps": 0, "loss": "l1_dssim"}).refine == \
        {"steps": 0, "loss": "l1_dssim"}


def test_refine_json_entries_with_densification():
    d = pr.DensifyConfig(until_step=3)
    kept = pr.RefineResult(torch.zeros(7, 14), torch.tensor([2.0, 1.0]), gaussians=[7, 9])
    assert pr.scene_report(kept, 1, "mse", d) == {"mse_before": 2.0, "mse_after": 1.0, "steps": 1,
                                                 "gaussians_before": 7, "gaussians_after": 9}
    copied = pr.RefineResult(torch.zeros(7, 14), torch.tensor([2.0]))
    assert pr.scene_report(copied, 0, "mse", d)["gaussians_after"] == 7
    report = pr.refine_report({"s": {}}, 4, {"rot": 0.5}, d)
    assert list(report) == ["steps", "lr", "scenes", "densify"] and report["lr"] == dict(LR, rot=0.5)
