"""GPU tests of the ablation and three-view presets end to end: each preset's whole encoder against the reference's
(tests/golden/presets_encoder_v1.npz, oracle/make_presets_golden.py), one training step per preset, the training
command line, bit-identical training and resume with three views, the validation step with three views, and the
evaluator on re10k_tiny.

re10k_tiny's scenes have 2 to 8 frames, so the training tests draw their views with the tiny bounded sampler
(TINY_SAMPLER of test_training_gpu.py; three context views for re10k_3_view) in place of the presets' 25 to 384
frame gaps."""
import json
from dataclasses import replace
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import make_presets_golden as mp
from oracle.make_backbone_golden import rel_err, seeded_state_dict
from pixelsplat_b200.data import ViewSamplerBoundedCfg, device_shim
from pixelsplat_b200.encoder.encoder_epipolar import EncoderEpipolar
from pixelsplat_b200.encoder.encoder_tail import EncoderEpipolarTail
from pixelsplat_b200.evaluation import Evaluator, Method, compute_metrics, load_checkpoint
from pixelsplat_b200.evaluation import presets as ev
from pixelsplat_b200.evaluation.checkpoint import read_checkpoint
from pixelsplat_b200.loss import compute_psnr, compute_ssim
from pixelsplat_b200.lpips import Lpips
from pixelsplat_b200.training import Trainer
from pixelsplat_b200.training import presets as tp
from pixelsplat_b200.training.trainer import VAL_METRICS, validation_rng
from tests import dataset_golden as dg
from tests import test_training_gpu as tt
from tests.test_training_gpu import deterministic  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
DEV = tt.DEV
GOLD = np.load(Path(__file__).resolve().parent / "golden" / "presets_encoder_v1.npz")
# test_backbone_gpu.py's floors for the TF32 attention kernels: outputs, and gradients back through attention
CEIL_OUT, CEIL_GRAD = 2e-3, 5e-2
TINY_SAMPLER_3 = ViewSamplerBoundedCfg(*mp.TINY_SAMPLER_3)
ABLATIONS = mp.NEW_PRESETS[:3]


def tiny(name: str) -> tp.TrainPreset:
    """The training preset with the tiny bounded sampler of its view count."""
    preset = tp.train_preset(name)
    return replace(preset, view_sampler=TINY_SAMPLER_3 if preset.view_sampler.num_context_views == 3
                   else tt.TINY_SAMPLER)


def train_cfg(name: str):
    return tp.dataset_cfg(tiny(name), dg.DATA)


def batches(name: str, n: int, seed: int = 5) -> list:
    """n host train batches (batch size 1) of the preset's tiny dataset."""
    torch.manual_seed(seed)
    out = []
    while len(out) < n:
        out += list(torch.utils.data.DataLoader(tp.make_train_dataset(train_cfg(name), None), batch_size=1,
                                                num_workers=0))
    return out[:n]


def model(name: str, full: bool = True, seed: int = 0):
    torch.manual_seed(seed)
    encoder, decoder = ev.build_model(tp.train_preset(name).model, train_cfg(name))
    if not full:
        encoder.backbone = tt.ConvBackbone()
    return encoder.to(DEV), decoder.to(DEV)


# ---- encoder parity with the reference


@pytest.fixture
def _no_tf32_convolutions():
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


@pytest.mark.parametrize("name,case", [(n, c) for n in mp.NEW_PRESETS for c in mp.cases(n)])
def test_encoder_matches_the_reference(name, case, _no_tf32_convolutions):
    import contextlib
    views = mp.num_views(name)
    enc = EncoderEpipolar(ev.encoder_cfg(name), num_context_views=views)
    enc.load_state_dict(seeded_state_dict(enc, mp.WEIGHT_SEED))
    enc = enc.to(DEV).eval()
    context = {k: v.to(DEV) for k, v in mp.inputs(views, torch.float32).items()}
    perm = case.split("_", 1)[1] if case.startswith("det_") else None
    torch.manual_seed(0)
    with mp.fixed_randperm(mp.PERMUTATIONS[perm]) if perm else contextlib.nullcontext():
        g = enc(context, global_step=0, deterministic=case.startswith("det"))
    out = mp.output_arrays(g)
    mp.weighted_sum(out, f"{name}/{case}/").backward()
    params = dict(enc.named_parameters())
    got = {k: v.detach().double().cpu().numpy() for k, v in out.items()}
    got.update({f"d_{k}": params[k].grad.reshape(-1)[:mp.PARAM_SLICE].double().cpu().numpy()
                for k in mp.GRAD_PARAMS if k in params})
    want = sorted(k[len(f"{name}/{case}/"):] for k in GOLD.files
                  if k.startswith(f"{name}/{case}/") and not k.endswith("_f32_err"))
    assert sorted(got) == want
    report = {}
    for k in want:
        key = f"{name}/{case}/{k}"
        ref = GOLD[key].astype(np.float64)
        assert got[k].shape == ref.shape, k
        err = rel_err(got[k], ref)
        bar = 4 * float(GOLD[key + "_f32_err"]) + (CEIL_GRAD if k.startswith("d_") else CEIL_OUT)
        report[k] = (err, bar)
    print(name, case, {k: f"{e:.1e}/{b:.1e}" for k, (e, b) in report.items()})
    assert all(e <= b for e, b in report.values()), report


# ---- training


@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    """One `Trainer.fit` step of each new preset's full encoder: {preset: (lines, checkpoint, initial, final)}."""
    out = {}
    for name in mp.NEW_PRESETS:
        encoder, decoder = model(name)
        initial = {k: v.detach().clone() for k, v in encoder.named_parameters()}
        t = Trainer(encoder, decoder, tp.make_losses(tiny(name), tt.seeded_lpips().to(DEV)), lr=1e-3,
                    warm_up_steps=1)
        loader = torch.utils.data.DataLoader(tp.make_train_dataset(train_cfg(name), None), batch_size=1,
                                             num_workers=0)
        path = tmp_path_factory.mktemp(name)
        lines = t.fit(loader, 1, path, checkpoint_every=1, log_every=1, log=None)
        final = {k: v.detach().clone() for k, v in encoder.named_parameters()}
        out[name] = (lines, path / "checkpoints" / f"epoch={t.epoch}-step=1.ckpt", initial, final)
        del t, encoder, decoder
    return out


@pytest.mark.parametrize("name", mp.NEW_PRESETS)
def test_one_training_step(name, trained):
    lines, ckpt, initial, final = trained[name]
    assert [l["step"] for l in lines] == [1]
    assert np.isfinite(lines[0]["total"]) and lines[0]["grad_norm"] > 0
    # the backbone runs DINO's ResNet-50 through layer3 only: layer4 gets no gradient
    unchanged = [k for k in initial if not k.startswith("backbone.resnet_backbone.model.layer4.")
                 and torch.equal(initial[k], final[k])]
    assert unchanged == []
    fresh, _ = ev.build_model(name, ev.dataset_cfg(dg.DATA, dg.DATA / "evaluation_index.json", preset=name))
    assert load_checkpoint(ckpt, fresh) == 1
    assert all(torch.equal(v.cpu(), final[k].cpu()) for k, v in fresh.named_parameters())


@pytest.mark.parametrize("name", ["re10k_3_view", "re10k_ablation_no_probabilistic_sampling"])
def test_command_line_runs_two_steps_and_resumes(name, tmp_path, monkeypatch):
    from pixelsplat_b200.training.__main__ import main
    monkeypatch.setattr(Lpips, "from_files", classmethod(lambda cls, *a, **k: tt.seeded_lpips()))
    monkeypatch.setitem(tp.TRAIN_PRESETS, name, tiny(name))
    common = ["--dataset-root", str(dg.DATA), "--preset", name, "--output", str(tmp_path), "--batch-size", "1",
              "--num-workers", "0", "--log-every", "1", "--overfit-to-scene", "ggg"]
    lines = main(common + ["--max-steps", "2"])
    assert [l["step"] for l in lines] == [1, 2] and all(np.isfinite(l["total"]) for l in lines)
    ckpt = tmp_path / "checkpoints" / "epoch=0-step=2.ckpt"
    state = read_checkpoint(ckpt)["state_dict"]
    assert ("encoder.epipolar_transformer.view_embeddings.weight" in state) == (name == "re10k_3_view")
    more = main(common + ["--max-steps", "3", "--resume", str(ckpt)])
    assert [l["step"] for l in more] == [3]


def test_three_view_runs_and_resume_are_bit_identical(deterministic, tmp_path):  # noqa: F811
    """The fixed-order epipolar backward at v = 3, with the view embeddings' permutation drawn each step."""
    bs = batches("re10k_3_view", 4)
    assert all(b["context"]["image"].shape[1] == 3 for b in bs)

    def trainer(**kw):
        return Trainer(*model("re10k_3_view", full=False), [tt.mse()], lr=tt.LR, warm_up_steps=tt.W, **kw)

    full = trainer()
    tt.run(full, bs[:2])
    full.save(tmp_path / "step2.ckpt")
    tt.run(full, bs[2:], seed=8)
    full.save(tmp_path / "a.ckpt")
    again = trainer()
    tt.run(again, bs[:2])
    tt.run(again, bs[2:], seed=8)
    again.save(tmp_path / "b.ckpt")
    resumed = trainer(step_tracker=None)
    resumed.resume(tmp_path / "step2.ckpt")
    tt.run(resumed, bs[2:], seed=8)
    resumed.save(tmp_path / "c.ckpt")

    a, b, c = (read_checkpoint(tmp_path / f"{n}.ckpt") for n in "abc")
    assert "encoder.epipolar_transformer.view_embeddings.weight" in a["state_dict"]
    for other in (b, c):
        assert other["global_step"] == a["global_step"] == 4
        assert tt.state_equal(a["state_dict"], other["state_dict"])
        sa, so = a["optimizer_states"][0]["state"], other["optimizer_states"][0]["state"]
        assert all(tt.state_equal(sa[i], so[i]) for i in sa)


def test_validation_step_with_three_views_equals_two_full_passes(deterministic, monkeypatch):  # noqa: F811
    """Both tails of the validation step see the one permutation its trunk draws; two full encoder passes that see
    that permutation give the same metrics and renders bit for bit."""
    cfg = tp.dataset_cfg(tiny("re10k_3_view"), dg.DATA)
    torch.manual_seed(3)
    batch = next(iter(torch.utils.data.DataLoader(tp.make_val_dataset(cfg, None), batch_size=1, num_workers=0)))
    batch = device_shim(batch, (256, 256), DEV)
    t = Trainer(*model("re10k_3_view"), [tt.mse()], lr=tt.LR, warm_up_steps=tt.W, lpips=tt.seeded_lpips())
    t.global_step = 7

    original, drawn, forced = torch.randperm, [], []

    def randperm(n, *args, **kwargs):
        p = original(n, *args, **kwargs)              # the same generator use as without the wrapper
        drawn.append(p.clone())
        return forced[0].clone() if forced else p

    monkeypatch.setattr(torch, "randperm", randperm)
    got = t.validation_step(batch)
    assert len(drawn) == 1 and len(got["context_index"]) == 3
    forced.append(drawn[0])

    encoder, decoder, lpips = t.encoder.eval(), t.decoder, t.lpips.eval()
    with torch.no_grad(), validation_rng(0, 7, DEV):
        b = encoder.get_data_shim()(batch)
        ctx, tgt = b["context"], b["target"]
        gt = tgt["image"][0]
        full, color, want = {}, {}, {}
        for tag in ("probabilistic", "deterministic"):
            full[tag] = encoder(ctx, 7, deterministic=tag == "deterministic")
            color[tag] = decoder.forward(full[tag], tgt["extrinsics"], tgt["intrinsics"], tgt["near"], tgt["far"],
                                         (256, 256)).color[0]
            want[f"psnr_{tag}"] = float(compute_psnr(gt, color[tag]).mean())
            want[f"ssim_{tag}"] = float(compute_ssim(gt, color[tag]).mean())
            want[f"lpips_{tag}"] = float(lpips(gt, color[tag], normalize=True)[:, 0, 0, 0].mean())
    with torch.no_grad(), validation_rng(0, 7, DEV):
        features, _ = encoder.trunk(ctx)
        shared = {tag: EncoderEpipolarTail.forward(encoder, features, ctx, 7, tag == "deterministic")
                  for tag in ("probabilistic", "deterministic")}
    assert len(drawn) == 4
    assert {k: got[k] for k in VAL_METRICS} == want and all(np.isfinite(got[k]) for k in VAL_METRICS)
    for tag in ("probabilistic", "deterministic"):
        assert torch.equal(got["images"][tag], color[tag]), tag
        for field in ("means", "covariances", "harmonics", "opacities"):
            assert torch.equal(getattr(shared[tag], field), getattr(full[tag], field)), (tag, field)


# ---- evaluation


def _test_loader(name: str):
    cfg = ev.dataset_cfg(dg.DATA, dg.DATA / "evaluation_index.json", dg.SHAPES["test"], preset=name)
    return cfg, torch.utils.data.DataLoader(ev.make_test_dataset(cfg), batch_size=1, num_workers=0)


def _reference_scenes(three_views: bool) -> list[str]:
    """The reference's test scenes on re10k_tiny.  With three context views its baseline check (which applies to
    two views only) no longer skips "eee", whose cameras share one position."""
    if not three_views:
        return [w["scene"] for w in dg.expected("test")]
    return [str(s) for s in np.load(dg.GOLDEN / "dataset_re10k_3view_v1.npz")["test/scene"]]


def test_evaluator_with_three_views(trained, tmp_path):
    cfg, loader = _test_loader("re10k_3_view")
    encoder, decoder = ev.build_model("re10k_3_view", cfg)
    assert load_checkpoint(trained["re10k_3_view"][1], encoder) == 1
    encoder, decoder = encoder.to(DEV).eval(), decoder.to(DEV)
    lp = tt.seeded_lpips().to(DEV)
    out = tmp_path / "three"
    res = Evaluator(encoder, decoder, out, lpips=lp).run(loader, (256, 256), keep_frames=True, log=None)
    assert [s.scene for s in res.scenes] == _reference_scenes(True) == ["aaa", "bbb", "eee"]
    for s in res.scenes:
        left, mid, right = s.context_index
        assert mid == (left + right) // 2
        for index in s.context_index:
            assert (out / s.scene / "context" / f"{index:0>6}.png").is_file()
        for i, index in enumerate(s.target_index):
            png = np.array(Image.open(out / s.scene / "color" / f"{index:0>6}.png"))
            assert np.array_equal(png, s.frames[i].cpu().numpy())
        assert all(np.isfinite(v) for v in s.metrics.values())
    assert len(json.loads((out / "benchmark.json").read_text())["encoder"]) == len(res.scenes)
    mc = compute_metrics([Method("Three views", "three", out)], _test_loader("re10k_3_view")[1], lpips=lp, log=None)
    assert mc.skipped == [] and list(mc.scenes) == [s.scene for s in res.scenes]
    for s in res.scenes:
        for k in ("psnr", "ssim", "lpips"):
            assert mc.scenes[s.scene][f"{k}_three"] == s.metrics[k], (s.scene, k)


@pytest.mark.parametrize("name", ABLATIONS)
def test_evaluator_with_each_ablation(name, trained):
    cfg, loader = _test_loader(name)
    encoder, decoder = ev.build_model(name, cfg)
    load_checkpoint(trained[name][1], encoder)
    res = Evaluator(encoder.to(DEV).eval(), decoder.to(DEV), lpips=tt.seeded_lpips().to(DEV)).run(
        loader, (256, 256), log=None)
    assert [s.scene for s in res.scenes] == _reference_scenes(False)
    assert all(len(s.context_index) == 2 and all(np.isfinite(v) for v in s.metrics.values()) for s in res.scenes)
