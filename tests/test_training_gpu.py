"""GPU tests of pixelsplat_b200.training on the tiny RE10k dataset of tests/dataset_golden.py (256 x 256, batch 1 or 2,
num_workers 0).

The bit-exact tests (two runs, resume) and the comparison with a plain-torch restatement run under
torch.use_deterministic_algorithms(True) with the preset encoder's transformer and tail behind a one-convolution
backbone: the preset's DINO + ResNet backbone upsamples its pyramid with F.interpolate, whose CUDA backward has no
deterministic implementation in torch.  The other tests (overfitting, the evaluator, the command line) run the full
preset encoder."""
import json
from dataclasses import replace

import pytest
import torch
from torch import nn

from oracle import lpips_oracle as lo
from pixelsplat_b200.data import ViewSamplerBoundedCfg, device_shim
from pixelsplat_b200.evaluation import Evaluator, load_checkpoint
from pixelsplat_b200.evaluation.checkpoint import read_checkpoint
from pixelsplat_b200.evaluation.presets import build_model
from pixelsplat_b200.loss import LossMse, LossMseCfg, LossMseCfgWrapper
from pixelsplat_b200.lpips import Lpips
from pixelsplat_b200.training import Trainer
from pixelsplat_b200.training import presets as tp
from tests import dataset_golden as dg

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
LR, W = 1e-3, 3
# re10k_tiny's scenes have 2 to 8 frames: the presets' context gap of 25 to 45 frames would skip them all
TINY_SAMPLER = ViewSamplerBoundedCfg("bounded", 2, 4, 2, 6, 0, 0, 2, 6)


class ConvBackbone(nn.Module):
    """A stand-in backbone without an upsample: one 3 x 3 convolution to the preset's 512 channels."""
    d_out = 512

    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(3, 512, 3, padding=1)

    def forward(self, context):
        image = context["image"]
        return self.conv(image.flatten(0, 1)).unflatten(0, image.shape[:2])


def batches(n, seed=5):
    """An explicit list of n train batches (host tensors, batch size 1)."""
    torch.manual_seed(seed)
    out = []
    while len(out) < n:
        out += list(torch.utils.data.DataLoader(dg.dataset("train"), batch_size=1, num_workers=0))
    return out[:n]


def model(full=False, seed=0):
    torch.manual_seed(seed)
    encoder, decoder = build_model("re10k", dg.dataset("train").cfg)
    if not full:
        encoder.backbone = ConvBackbone()
    return encoder.to(DEV), decoder.to(DEV)


def mse():
    return LossMse(LossMseCfgWrapper(LossMseCfg(1.0)))


def trainer(full=False, fused=None, **kw):
    return Trainer(*model(full), [mse()], lr=LR, warm_up_steps=W, fused_mse=fused, **kw)


def run(t, bs, seed=7):
    """Steps `t` over the batch list with torch's generators seeded; returns the per-step host values."""
    torch.manual_seed(seed)
    out = []
    for b in bs:
        t.training_step(device_shim(b, (256, 256), DEV))
        out.append(t.read_last())
    return out


@pytest.fixture
def deterministic(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(False)


def state_equal(a: dict, b: dict) -> bool:
    return a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def test_four_steps_equal_a_plain_torch_restatement(deterministic):
    bs = batches(4)
    t = trainer(fused=False)
    init = [p.detach().clone() for p in t.encoder.parameters()]
    ours = run(t, bs)

    encoder, decoder = model()
    params = list(encoder.parameters())
    adam = torch.optim.Adam(params, lr=LR)
    sched = torch.optim.lr_scheduler.LinearLR(adam, 1 / W, 1, total_iters=W)
    shim, loss_fn = encoder.get_data_shim(), mse()
    torch.manual_seed(7)
    for step, b in enumerate(bs):
        b = shim(device_shim(b, (256, 256), DEV))
        tg = b["target"]
        adam.zero_grad()
        gaussians = encoder(b["context"], step, False)
        out = decoder.forward(gaussians, tg["extrinsics"], tg["intrinsics"], tg["near"], tg["far"], (256, 256))
        loss = loss_fn(out, b, gaussians, step)
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(params, 0.5)
        adam.step()
        sched.step()
        assert ours[step]["total"] == pytest.approx(float(loss.detach()), rel=1e-4)
        assert ours[step]["mse"] == pytest.approx(float(loss.detach()), rel=1e-4)
        assert ours[step]["grad_norm"] == pytest.approx(float(norm), rel=1e-3)
    worst = 0.0
    for p0, a, b in zip(init, t.encoder.parameters(), params):
        moved = float((b - p0).detach().norm())
        err = float((a - b).detach().norm())
        worst = max(worst, err / moved if moved > 0 else (0.0 if err == 0 else float("inf")))
    print(f"trainer vs torch restatement after 4 steps: worst ||ours - torch|| / ||torch - init|| = {worst:.2e}")
    assert worst <= 0.02                                    # of the distance each parameter moved; 3.6e-3 on an H100


def test_fused_mse_route_equals_the_rendered_image_route(deterministic):
    bs = batches(2)
    a, b = trainer(fused=True), trainer(fused=False)
    assert a.fused_mse and not b.fused_mse
    init = [p.detach().clone() for p in a.encoder.parameters()]
    la, lb = run(a, bs), run(b, bs)
    for x, y in zip(la, lb):
        assert x["mse"] == pytest.approx(y["mse"], rel=1e-4) and x["psnr"] == pytest.approx(y["psnr"], abs=1e-3)
    num = sum(float((p - q).detach().norm()) ** 2 for p, q in zip(a.encoder.parameters(), b.encoder.parameters())) ** 0.5
    den = sum(float((q - p0).detach().norm()) ** 2 for q, p0 in zip(b.encoder.parameters(), init)) ** 0.5
    print(f"fused vs rendered route after 2 steps: ||difference|| / ||movement|| = {num / den:.2e}")
    assert num <= 1e-3 * den                                # identical bits on an H100


def test_deterministic_runs_and_resume_are_bit_identical(deterministic, tmp_path):
    bs = batches(4)
    full = trainer()
    run(full, bs[:2])
    full.save(tmp_path / "step2.ckpt")
    run(full, bs[2:], seed=8)
    full.save(tmp_path / "a.ckpt")

    again = trainer()
    run(again, bs[:2])
    again.save(tmp_path / "again2.ckpt")                    # saving consumes no random numbers
    run(again, bs[2:], seed=8)
    again.save(tmp_path / "b.ckpt")

    resumed = trainer(step_tracker=None)
    with torch.no_grad():
        for p in resumed.encoder.parameters():
            p.add_(1.0)                                     # whatever it held is replaced
    resumed.resume(tmp_path / "step2.ckpt")
    assert resumed.global_step == 2 and resumed.optimizer.lr() == full.optimizer.base_lr * (1 / W + (1 - 1 / W) * 2 / W)
    assert int(resumed.optimizer.step_counter) == 2
    run(resumed, bs[2:], seed=8)
    resumed.save(tmp_path / "c.ckpt")

    a, b, c = (read_checkpoint(tmp_path / f"{n}.ckpt") for n in "abc")
    for other in (b, c):
        assert other["global_step"] == a["global_step"] == 4
        assert state_equal(a["state_dict"], other["state_dict"])
        sa, so = a["optimizer_states"][0]["state"], other["optimizer_states"][0]["state"]
        assert all(state_equal(sa[i], so[i]) for i in sa)
        assert a["optimizer_states"][0]["param_groups"] == other["optimizer_states"][0]["param_groups"]
        assert a["lr_schedulers"] == other["lr_schedulers"]


def seeded_lpips():
    lp = Lpips()
    lp.load_state_dict(lo.random_state_dict(0))
    return lp


def test_overfitting_lowers_the_mse_and_the_checkpoint_feeds_the_evaluator(tmp_path):
    preset = tp.train_preset("re10k")
    scene = "ggg"
    cfg = tp.dataset_cfg(replace(preset, view_sampler=TINY_SAMPLER), dg.DATA, overfit_to_scene=scene)
    torch.manual_seed(0)
    encoder, decoder = build_model("re10k", cfg)
    t = Trainer(encoder.to(DEV), decoder.to(DEV), [mse()], lr=5e-4, warm_up_steps=5)
    loader = torch.utils.data.DataLoader(tp.make_train_dataset(cfg, None), batch_size=2, num_workers=0)
    lines = t.fit(loader, 40, tmp_path, checkpoint_every=40, log_every=1, log=None)
    assert [l["step"] for l in lines] == list(range(1, 41))
    first, last = (sum(l["mse"] for l in part) / 5 for part in (lines[:5], lines[-5:]))
    print(f"overfit to {scene}: mean MSE of steps 1-5 {first:.4f}, of steps 36-40 {last:.4f}; "
          f"phase_ms of step 40 {lines[-1]['phase_ms']}")
    assert last < 0.5 * first                                # a sanity bound, not a benchmark (0.251 -> 0.028 on an H100)
    assert all(l["grad_norm"] > 0 and l["lr"] > 0 and l["scenes_per_s"] > 0 for l in lines)
    assert [json.loads(s)["step"] for s in (tmp_path / "log.jsonl").read_text().splitlines()] == list(range(1, 41))

    ckpt = tmp_path / "checkpoints" / f"epoch={t.epoch}-step=40.ckpt"
    fresh, dec = build_model("re10k", dg.dataset("test").cfg)
    assert load_checkpoint(ckpt, fresh) == 40
    test_loader = torch.utils.data.DataLoader(dg.dataset("test"), batch_size=1, num_workers=0)
    res = Evaluator(fresh.to(DEV).eval(), dec.to(DEV), lpips=seeded_lpips().to(DEV)).run(test_loader, (256, 256), log=None)
    assert res.scenes and all(v == v and abs(v) != float("inf") for v in res.mean.values())


def test_command_line_runs_two_steps_and_resumes(tmp_path, monkeypatch, capsys):
    from pixelsplat_b200.training.__main__ import main
    monkeypatch.setattr(Lpips, "from_files", classmethod(lambda cls, *a, **k: seeded_lpips()))
    monkeypatch.setitem(tp.TRAIN_PRESETS, "re10k", replace(tp.train_preset("re10k"), view_sampler=TINY_SAMPLER))
    common = ["--dataset-root", str(dg.DATA), "--preset", "re10k", "--output", str(tmp_path), "--batch-size", "1",
              "--num-workers", "0", "--log-every", "1", "--overfit-to-scene", "ggg"]
    lines = main(common + ["--max-steps", "2"])
    assert [l["step"] for l in lines] == [1, 2] and {"mse", "lpips", "total", "psnr", "grad_norm", "lr"} <= set(lines[0])
    assert lines[0]["lpips"] == 0.0                          # LossLpips applies after step 150 000
    assert "random initialisation" in capsys.readouterr().out
    ckpt = tmp_path / "checkpoints" / "epoch=0-step=2.ckpt"
    assert ckpt.is_file() and len((tmp_path / "log.jsonl").read_text().splitlines()) == 2
    more = main(common + ["--max-steps", "3", "--resume", str(ckpt)])
    assert [l["step"] for l in more] == [3]
    assert more[0]["lr"] == pytest.approx(1.5e-4 * (1 / 2000 + (1 - 1 / 2000) * 2 / 2000), rel=1e-9)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_end_a_step_with_identical_parameters(tmp_path):
    import subprocess
    import sys
    script = tmp_path / "two_ranks.py"
    script.write_text(f"""
import sys, torch, torch.distributed as dist
sys.path.insert(0, {str(dg.GOLDEN.parents[1])!r})
from pixelsplat_b200 import parallel
from tests import test_training_gpu as tt
rank, world, local = parallel.init_distributed()
torch.cuda.set_device(local)
tt.DEV = torch.device("cuda", local)
t = tt.Trainer(*tt.model(seed=rank), [tt.mse()], lr=tt.LR, warm_up_steps=tt.W)
tt.run(t, tt.batches(2, seed=5 + rank), seed=7 + rank)
flat = torch.cat([p.detach().reshape(-1) for p in t.encoder.parameters()])
both = [torch.empty_like(flat) for _ in range(world)]
dist.all_gather(both, flat)
assert torch.equal(both[0], both[1]), "ranks disagree"
dist.destroy_process_group()
""")
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2", "--master-addr",
                    "127.0.0.1", str(script)], check=True, timeout=600)
