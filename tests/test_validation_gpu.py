"""GPU tests of the training's validation step and its place in `Trainer.fit` and the command line, on the tiny RE10k
dataset of tests/dataset_golden.py (256 x 256, one scene per validation, 2 context views and 4 targets).

The step's metrics, renders and Gaussians are compared bit for bit with two full encoder passes under
torch.use_deterministic_algorithms(True), with the preset encoder (DINO + ResNet-50 backbone: its forward is
deterministic).  The training comparisons (validation on against off, resume) take gradients, so they use the
one-convolution backbone of test_training_gpu.py, as its bit-exact tests do."""
import json
from dataclasses import replace

import numpy as np
import pytest
import torch

from pixelsplat_b200.data import device_shim
from pixelsplat_b200.encoder.encoder_tail import EncoderEpipolarTail
from pixelsplat_b200.evaluation.image_io import quantise, read_frame
from pixelsplat_b200.evaluation.checkpoint import read_checkpoint
from pixelsplat_b200.loss import compute_psnr, compute_ssim
from pixelsplat_b200.lpips import Lpips
from pixelsplat_b200.training import Trainer
from pixelsplat_b200.training import presets as tp
from pixelsplat_b200.training.trainer import VAL_METRICS, comparison_layout, validation_rng
from tests import dataset_golden as dg
from tests import test_training_gpu as tt
from tests.test_training_gpu import deterministic  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
DEV = tt.DEV


def val_batches(n, seed=3):
    """n host batches of one scene from the stage-"val" dataset (the test split, 4 targets)."""
    cfg = tp.dataset_cfg(replace(tp.train_preset("re10k"), view_sampler=tt.TINY_SAMPLER), dg.DATA)
    torch.manual_seed(seed)
    out = []
    while len(out) < n:
        out += list(torch.utils.data.DataLoader(tp.make_val_dataset(cfg, None), batch_size=1, num_workers=0))
    return out[:n]


def trainer(full=False):
    return Trainer(*tt.model(full), [tt.mse()], lr=tt.LR, warm_up_steps=tt.W, lpips=tt.seeded_lpips())


def test_step_equals_two_full_encoder_passes(deterministic):  # noqa: F811
    t = trainer(full=True)
    t.global_step = 7                                       # the step reaches the tail's opacity schedule
    batch = device_shim(val_batches(1)[0], (256, 256), DEV)
    got = t.validation_step(batch)
    assert got["step"] == 7 and got["scene"] == batch["scene"][0] and len(got["context_index"]) == 2

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

    print("validation step:", {k: got[k] for k in VAL_METRICS}, got["phase_ms"])
    assert {k: got[k] for k in VAL_METRICS} == want
    assert all(np.isfinite(got[k]) for k in VAL_METRICS)
    for tag in ("probabilistic", "deterministic"):
        assert torch.equal(got["images"][tag], color[tag]), tag
        for field in ("means", "covariances", "harmonics", "opacities"):
            assert torch.equal(getattr(shared[tag], field), getattr(full[tag], field)), (tag, field)
    assert torch.equal(got["images"]["target"], gt) and torch.equal(got["images"]["context"], ctx["image"][0])
    # the two encodings differ (the probabilistic tail samples its depths)
    assert not torch.equal(full["probabilistic"].means, full["deterministic"].means)


def test_step_changes_no_training_state():
    t = trainer(full=True)
    tt.run(t, tt.batches(1))                                # non-zero moments, BatchNorm statistics that moved
    batch = device_shim(val_batches(1)[0], (256, 256), DEV)
    t.encoder.train()
    t.encoder.backbone.eval()                               # a mixed tree of modes comes back as it was
    modes = [m.training for m in t.encoder.modules()]
    state = {k: v.clone() for k, v in t.encoder.state_dict().items()}
    assert any("running_mean" in k for k in state)
    opt = t.optimizer.state_dict()
    moments = {i: {k: v.clone() for k, v in s.items()} for i, s in opt["state"].items()}
    counter = t.optimizer.step_counter.clone()
    cpu, cuda = torch.get_rng_state(), torch.cuda.get_rng_state(DEV)

    t.validation_step(batch)
    torch.cuda.synchronize()
    assert [m.training for m in t.encoder.modules()] == modes
    assert tt.state_equal(state, t.encoder.state_dict())
    after = t.optimizer.state_dict()["state"]
    assert all(tt.state_equal(moments[i], after[i]) for i in moments)
    assert torch.equal(counter, t.optimizer.step_counter)
    assert torch.equal(cpu, torch.get_rng_state()) and torch.equal(cuda, torch.cuda.get_rng_state(DEV))
    assert t.global_step == 1

    # the comparison is sensitive: under no_grad in train mode the BatchNorm statistics move
    t.encoder.train()
    with torch.no_grad():
        t.encoder.trunk(t.data_shim(batch)["context"])
    assert not tt.state_equal(state, t.encoder.state_dict())


def fit(output, bs, vs, val_every, max_steps=4, t=None, capture=None, seed=7):
    """`Trainer.fit` over the batch list, checkpoints every 2 steps; `seed` None keeps the generators as they are
    (a resumed trainer's come from its checkpoint)."""
    t = t if t is not None else trainer()
    if capture is not None:
        step = t.validation_step
        t.validation_step = lambda b: capture.append(step(b)) or capture[-1]
    if seed is not None:
        torch.manual_seed(seed)
    t.fit(bs, max_steps, output, checkpoint_every=2, log_every=1, log=None, validation=vs, val_every=val_every)
    return t


def log_lines(path):
    timing = ("phase_ms", "scenes_per_s")
    return [{k: v for k, v in json.loads(s).items() if k not in timing} for s in path.read_text().splitlines()]


def test_validation_leaves_the_training_bits_and_the_resume_unchanged(deterministic, tmp_path):  # noqa: F811
    bs, vs = tt.batches(4), val_batches(2)
    off = fit(tmp_path / "off", bs, None, 0)
    on = fit(tmp_path / "on", bs, vs, 2)
    assert tt.state_equal(off.encoder.state_dict(), on.encoder.state_dict())
    assert log_lines(tmp_path / "off" / "log.jsonl") == log_lines(tmp_path / "on" / "log.jsonl")

    resumed = trainer()
    resumed.resume(tmp_path / "on" / "checkpoints" / "epoch=0-step=2.ckpt")
    fit(tmp_path / "resumed", bs[2:], vs, 2, t=resumed, seed=None)
    a = read_checkpoint(tmp_path / "on" / "checkpoints" / "epoch=0-step=4.ckpt")
    c = read_checkpoint(tmp_path / "resumed" / "checkpoints" / "epoch=0-step=4.ckpt")
    assert tt.state_equal(a["state_dict"], c["state_dict"])
    assert all(tt.state_equal(a["optimizer_states"][0]["state"][i], c["optimizer_states"][0]["state"][i])
               for i in a["optimizer_states"][0]["state"])


def test_fit_writes_one_line_and_one_comparison_image_per_validation(tmp_path):
    bs, vs, results = tt.batches(4), val_batches(2), []
    fit(tmp_path, bs, vs, 2, capture=results)
    lines = [json.loads(s) for s in (tmp_path / "validation.jsonl").read_text().splitlines()]
    assert [l["step"] for l in lines] == [0, 2, 4] == [r["step"] for r in results]
    # one iterator over the two batches, restarted when exhausted
    assert [l["scene"] for l in lines] == [vs[0]["scene"][0], vs[1]["scene"][0], vs[0]["scene"][0]]
    for line, r in zip(lines, results):
        assert set(line) == {"step", "scene", "context_index", *VAL_METRICS, "ms"}
        assert all(np.isfinite(line[k]) for k in VAL_METRICS) and line["ms"] > 0
        assert {k: line[k] for k in VAL_METRICS} == {k: r[k] for k in VAL_METRICS}
        im = r["images"]
        want = quantise(comparison_layout(im["context"], im["target"], im["probabilistic"], im["deterministic"]))
        got = read_frame(tmp_path / "validation" / f"comparison_{line['step']:0>6}.png")
        assert got.shape == (8 + 4 * 256 + 3 * 8 + 8, 8 + 4 * 256 + 3 * 8 + 8, 3)
        assert np.array_equal(got, want.cpu().numpy())
    assert sorted(p.name for p in (tmp_path / "validation").iterdir()) == \
        [f"comparison_{s:0>6}.png" for s in (0, 2, 4)]
    assert [json.loads(s)["step"] for s in (tmp_path / "log.jsonl").read_text().splitlines()] == [1, 2, 3, 4]


def test_command_line_validates_before_the_first_step_and_after_resuming(tmp_path, monkeypatch):
    from pixelsplat_b200.training.__main__ import main
    monkeypatch.setattr(Lpips, "from_files", classmethod(lambda cls, *a, **k: tt.seeded_lpips()))
    monkeypatch.setitem(tp.TRAIN_PRESETS, "re10k", replace(tp.train_preset("re10k"), view_sampler=tt.TINY_SAMPLER))
    common = ["--dataset-root", str(dg.DATA), "--preset", "re10k", "--output", str(tmp_path), "--batch-size", "1",
              "--num-workers", "0", "--log-every", "1", "--val-every", "1"]
    lines = main(common + ["--max-steps", "2"])
    assert [l["step"] for l in lines] == [1, 2]
    read = lambda: [json.loads(s) for s in (tmp_path / "validation.jsonl").read_text().splitlines()]
    assert [l["step"] for l in read()] == [0, 1, 2]
    assert len((tmp_path / "log.jsonl").read_text().splitlines()) == 2
    more = main(common + ["--max-steps", "3", "--resume", str(tmp_path / "checkpoints" / "epoch=0-step=2.ckpt")])
    assert [l["step"] for l in more] == [3]
    val = read()
    assert [l["step"] for l in val] == [0, 1, 2, 2, 3]
    assert all(np.isfinite(l[k]) for l in val for k in VAL_METRICS)
    # the resumed run's sanity check rewrites comparison_000002.png
    assert sorted(p.name for p in (tmp_path / "validation").iterdir()) == \
        [f"comparison_{s:0>6}.png" for s in (0, 1, 2, 3)]
